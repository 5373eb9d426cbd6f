"""CPU tests of the compiled step program (`pycolab_b200.compiler`, csrc/compiled.cu).

  - what the compiler accepts and refuses, with the source line in the message;
  - with the reference present, the oracle interpreter (oracle/compiled.py) running the
    compiled words of its own classics examples reproduces their goldens (the games of
    tests/compiled_games.py replay theirs in test_registered_goldens.py);
  - pcl_bind_code's checks, on handles that never reach a device;
  - the kernel keeps its operand stack out of local memory.
"""

import ctypes as C
import os
import sys

import numpy as np
import pytest

import boundary_sweep
import example_games as eg
import golden_cases as gc
import refdriver
import registered_games as rg
import trajectory as tj
from oracle import compiled as ocompiled
from pycolab_b200 import _lib, compiler, lowering
from pycolab_b200 import things as b_things
from pycolab_b200.errors import NotLoweredError

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope='module')
def games():
  yield from rg.registered('compiled_games.py')


def test_registered_class_wins_and_unregistered_is_refused(games):
  engine = games.make_coins(0)
  assert lowering.lower(engine).program == _lib.PROG_COMPILED
  compiler.unregister(games.CoinDrape)
  try:
    with pytest.raises(NotLoweredError, match='CoinDrape'):
      lowering.lower(games.make_coins(0))
  finally:
    compiler.register(games.CoinDrape)


def test_subclass_overriding_update_is_not_compiled(games):
  class Edited(games.CoinDrape):
    def update(self, actions, board, layers, backdrop, things, the_plot):
      pass
  assert compiler.registered(games.CoinDrape) is not None
  assert compiler.registered(Edited) is None

  class Plain(games.CoinDrape):
    pass
  assert compiler.registered(Plain) is compiler.registered(games.CoinDrape)


def test_missing_plot_key_and_float_register_are_refused(games):
  engine = games.make_coins(0)
  del engine.the_plot['countdown']
  with pytest.raises(NotLoweredError, match="the_plot\\['countdown'\\]"):
    lowering.lower(engine)
  engine = games.make_coins(0)
  engine.things['P'].bumps = 0.5
  with pytest.raises(NotLoweredError, match='bumps'):
    lowering.lower(engine)


def test_float_rewards_select_the_float64_output(games):
  spec = lowering.lower(games.make_lava(0)).make_spec(True)
  assert spec.program_arg[0] == 1
  spec = lowering.lower(games.make_coins(0)).make_spec(True)
  assert spec.program_arg[0] == 0


# ---------------------------------------------------------------- the subset --

# Each refused construct, as a walker whose update() has it on the marked line.
def _loop(self, actions, board, layers, backdrop, things, the_plot):
  for _ in range(3):                                  # REFUSED
    pass


def _float_math(self, actions, board, layers, backdrop, things, the_plot):
  self.n = self.n * 0.5                               # REFUSED


def _other_call(self, actions, board, layers, backdrop, things, the_plot):
  the_plot.log('hello')                               # REFUSED


def _ordering_on_actions(self, actions, board, layers, backdrop, things, the_plot):
  if actions < 2:                                     # REFUSED
    self._north(board, the_plot)


def _slice(self, actions, board, layers, backdrop, things, the_plot):
  self.n = board[1:3, 2]                              # REFUSED


def _z_order(self, actions, board, layers, backdrop, things, the_plot):
  the_plot.change_z_order('P', None)                  # REFUSED


def _random(self, actions, board, layers, backdrop, things, the_plot):
  self.n = random.randint(0, 3)                       # REFUSED  # noqa: F821


def _comprehension(self, actions, board, layers, backdrop, things, the_plot):
  self.n = sum([1 for _ in 'ab'])                     # REFUSED


def _cell_arithmetic_string(self, actions, board, layers, backdrop, things, the_plot):
  if board[1, 1] in '#@':                             # REFUSED
    pass


def _float_reward_expression(self, actions, board, layers, backdrop, things, the_plot):
  the_plot.add_reward(self.n * 0.5)                   # REFUSED


def _prefab_state(self, actions, board, layers, backdrop, things, the_plot):
  self._virtual_row = 3                               # REFUSED


def _position_truth(self, actions, board, layers, backdrop, things, the_plot):
  if self.position:                                   # REFUSED
    pass


REFUSED = [(_loop, 'For'), (_float_math, 'literal 0.5'), (_other_call, 'the_plot.log()'),
           (_ordering_on_actions, 'ordering comparison'), (_slice, 'Slice'),
           (_z_order, 'the_plot.change_z_order()'), (_random, 'random.randint()'),
           (_comprehension, 'the call sum()'), (_cell_arithmetic_string, 'string on a number'),
           (_float_reward_expression, 'literal 0.5'), (_prefab_state, '_virtual_row'),
           (_position_truth, 'position as a truth value')]


@pytest.mark.parametrize('update,what', REFUSED, ids=[u.__name__ for u, _ in REFUSED])
def test_refused_construct_names_class_line_and_construct(update, what):
  msg = rg.assert_refused(rg.walker(update), what)
  assert '# REFUSED' in msg, msg                  # the source line itself


def _accepted(self, actions, board, layers, backdrop, things, the_plot):
  """A docstring."""
  del layers
  pos = self.virtual_position
  if actions in (0, 1) and not (self.n >= 3 or self.n < -3):
    self._northeast(board, the_plot)
  elif actions is not None and actions != 7:
    moved = self._southwest(board, the_plot)
    if moved is None:
      self.n -= -7 // 2 % 3
  if pos == (self.position.row, self.position[1]) and 0 <= self.n < 4 < 5:
    the_plot['k'] = int(self.visible) + ord('a') - the_plot.frame
  if chr(board[pos]) in ('#', '@') or backdrop.curtain[-1, -1] == ord(' '):
    self._teleport((self.corner.row - 1, 0))
  the_plot.change_default_discount(0.9)
  the_plot.add_reward(3 if self.n else -1)
  return


def test_accepted_constructs_compile():
  comp = compiler.compile_class(rg.walker(_accepted))
  assert comp.attrs == ['n'] and comp.keys == ['k'] and not comp.float_reward
  ops = {ins[0] for ins in comp.ir}
  assert {'MOVE', 'TELEPORT', 'IN', 'EQ2', 'FLOORDIV', 'MOD', 'BACKDROP', 'BOARD', 'FRAME',
          'DISCOUNT', 'REWARD'} <= ops


def test_drape_only_and_sprite_only_constructs_are_checked():
  def fill(self, actions, board, layers, backdrop, things, the_plot):
    self.curtain[:] = True
  with pytest.raises(NotLoweredError, match='curtain write in a sprite class'):
    compiler.compile_class(rg.walker(fill))

  def move(self, actions, board, layers, backdrop, things, the_plot):
    self._north(board, the_plot)
  with pytest.raises(NotLoweredError, match='_north in a drape class'):
    compiler.compile_class(type('D', (b_things.Drape,), {'update': move}))


# ------------------------------------------------------------- the classics --

needs_ref = pytest.mark.skipif(not refdriver.available(), reason='/root/reference not present')


@needs_ref
@pytest.mark.parametrize('name', gc.names('classic_'))
def test_reference_classics_compile_and_match_golden(name):
  g = gc.load(name)
  kind, art = bytes(g['kind']).decode(), tj.u8_to_art(g['art'])
  mod = rg.load(os.path.join(refdriver.REFERENCE_ROOT, 'pycolab', 'examples', 'classics',
                             kind + '.py'))
  compiler.register(mod.PlayerSprite)
  try:
    saved, mod.GAME_ART = mod.GAME_ART, art
    try:
      lowered = lowering.lower(mod.make_game())
    finally:
      mod.GAME_ART = saved
  finally:
    compiler.unregister(mod.PlayerSprite)
  assert lowered.program == _lib.PROG_COMPILED
  assert lowered.float_reward and lowered.reward_type is float
  eg.assert_replays('oracle', name, make_env=lambda: ocompiled.make_world(lowered))


# ------------------------------------------------------------ pcl_bind_code --

def _outputs():
  f = boundary_sweep.FAKE
  return _lib.Outputs(f, f, f, f, f, f)


def test_bind_code_checks(games):
  lib = _lib.load()
  lowered = lowering.lower(games.make_coins(0))
  spec = lowered.make_spec(True)
  code = lowered.code.copy()
  h = rg.handle(lib, spec)
  try:
    # step and reset before any code is bound
    assert lib.pcl_bind_state(h, C.byref(boundary_sweep._full_state())) == _lib.OK
    out = _outputs()
    assert lib.pcl_step(h, boundary_sweep.FAKE, C.byref(out), None) == _lib.ERR_UNBOUND
    assert lib.pcl_reset(h, None, C.byref(out), None) == _lib.ERR_UNBOUND
    assert rg.bind(lib, h, code) == _lib.OK
    n_ent = code[0]
    body = 1 + n_ent
    first = code[1]                    # the player's update (sprite 0)
    op = lambda name: _lib.OP[name]

    def mutated(at, value):
      c = code.copy()
      c[at] = value
      return c
    # the first instruction of the player's code, and of the drape's
    assert code[first] == op('ACTION')
    cases = {
        'bad opcode': mutated(first, 99),
        'negative opcode': mutated(first, -1),
        'entity count': mutated(0, n_ent + 1),
        'entry out of range': mutated(1, len(code)),
        'entry into the header': mutated(1, 0),
        'oversize': np.zeros(_lib.MAX_CODE_WORDS + 1, dtype=np.int32),
        'empty': code[:body],
    }
    pc = ocompiled.instructions(code, first, code[2])
    jz = [i for i in pc if code[i] == op('JZ')][0]
    cases['backward jump'] = mutated(jz + 1, jz)
    cases['jump out of the function'] = mutated(jz + 1, len(code) + 5)
    cases['jump into an operand'] = mutated(jz + 1, jz + 1)
    getr = [i for i in ocompiled.instructions(code, code[2], code[3]) if code[i] == op('GETR')][0]
    cases['register out of range'] = mutated(getr + 1, 3)     # sprites have 3 registers
    field = [i for i in ocompiled.instructions(code, code[3], len(code))
             if code[i] == op('FIELD')][0]
    cases['entity out of range'] = mutated(field + 1, 2)      # drape 'c' is entity 2
    cases['sprite entity past the end'] = mutated(field + 1, 7)
    load = ocompiled.instructions(code, first, code[2])
    store = [i for i in load if code[i] == op('STORE')][0]
    cases['local out of range'] = mutated(store + 1, _lib.CODE_LOCALS)
    cases['no RET at the end'] = mutated(len(code) - 1, op('POP'))
    cases['stack underflow'] = mutated(first, op('POP'))
    for label, words in cases.items():
      assert rg.bind(lib, h, words) == _lib.ERR_INVALID, label
    assert lib.pcl_bind_code(h, None, 4) == _lib.ERR_INVALID
  finally:
    lib.pcl_destroy(h)


def test_bind_code_is_refused_by_other_programs():
  lib = _lib.load()
  from pycolab_b200.games.classics import four_rooms
  h = rg.handle(lib, lowering.lower(four_rooms.make_game()).make_spec(True))
  try:
    assert rg.bind(lib, h, [1, 2, 0]) == _lib.ERR_UNSUPPORTED
  finally:
    lib.pcl_destroy(h)


# ------------------------------------------------------------- the kernel --

def test_compiled_step_keeps_its_stack_in_shared_memory():
  import test_kernel_resources as kr
  if kr._cuobjdump() is None:
    pytest.skip('cuobjdump not found')
  kernels = {n: u for n, u in kr._resource_usage(_lib.LIB_PATH).items() if 'compiled_step' in n}
  assert kernels, 'no compiled_step in %s' % _lib.LIB_PATH
  for name, u in kernels.items():
    assert u['STACK'] == 0, (name, u)


@needs_ref
def test_bench_player_compiles_like_the_reference_four_rooms():
  """tools/compiled_bench.py times the same words the reference's own class compiles to."""
  sys.path.insert(0, os.path.join(os.path.dirname(HERE), 'tools'))
  try:
    import compiled_bench
  finally:
    sys.path.pop(0)
  mod = rg.load(os.path.join(refdriver.REFERENCE_ROOT, 'pycolab', 'examples', 'classics',
                             'four_rooms.py'))
  theirs = compiler.compile_class(mod.PlayerSprite)
  ours = compiler.compile_class(compiled_bench.FourRoomsPlayer)
  link = lambda c: compiler.link({'P': c}, 'P', '', 13, 13, []).tolist()
  assert link(theirs) == link(ours)
