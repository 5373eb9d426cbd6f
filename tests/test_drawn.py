"""CPU tests of draws from the global generators in compiled update() code
(`pycolab_b200.compiler`, include/pcl.h PCL_OP_RANDINT / RANDCMP / PICK).

  - the draw forms the compiler accepts, through aliased imports too, and the forms it
    refuses, with the class, the source line and the construct;
  - the oracle's restatement of the draws equals NumPy's RandomState and Python's Random
    in value and in the words consumed, over the edge ranges and across a twist;
  - pcl_create / pcl_bind_state / pcl_bind_code refuse bad RNG slots, on handles that never
    reach a device;
  - games without draws lower as before.
"""

import ctypes as C
import random

import numpy as np
import pytest

import boundary_sweep
import registered_games as rg
from oracle import compiled as ocompiled
from pycolab_b200 import _lib, compiler, lowering

SEQ = (1, 2, 3)


@pytest.fixture(scope='module')
def games():
  yield from rg.registered('drawn_games.py')


# ------------------------------------------------------------------ the subset --

def test_accepted_draws_compile_through_aliases(games):
  streams = {k.__name__: compiler.registered(k).streams for k in games.CLASSES}
  assert streams == {'Player': ['numpy', 'python'], 'NumpyMonster': ['numpy'],
                     'PythonMonster': ['python'], 'Fruit': ['python', 'numpy'],
                     'Edges': ['numpy', 'python'], 'Thresholds': ['numpy', 'python'],
                     'EmptyRange': ['numpy', 'python']}
  ops = {ins[0] for k in games.CLASSES for ins in compiler.registered(k).ir}
  assert {'RANDINT', 'RANDCMP', 'PICK'} <= ops
  lowered = lowering.lower(games.make_monsters(0))
  assert lowered.rng_streams == ('numpy', 'python')
  assert lowered.rng_from_globals and lowered.program_arg[1] == 2
  # `from random import randint` and `from numpy import random as npr` in Fruit
  fruit = compiler.registered(games.Fruit).ir
  rules = [ins[2] for ins in fruit if ins[0] == 'RANDINT']
  assert rules == [_lib.RAND_PYTHON_CLOSED, _lib.RAND_NUMPY]


def test_float_draw_on_either_side_of_the_comparison():
  def update(self, actions, board, layers, backdrop, things, the_plot):
    if 0.25 > np.random.rand():
      self.n = 1
    if random.random() != -1:
      self.n = 2
  comp = compiler.compile_class(rg.walker(update))
  cmps = [ins for ins in comp.ir if ins[0] == 'RANDCMP']
  assert [c[2] for c in cmps] == [2, 1]          # 0.25 > x as x < 0.25; x != -1
  assert [c[1] for c in cmps] == [('rng', 'numpy'), ('rng', 'python')]


# Each refused draw, as a walker whose update() has it on the marked line.
def _size(self, actions, board, layers, backdrop, things, the_plot):
  self.n = np.random.randint(3, size=1)                # REFUSED


def _dtype(self, actions, board, layers, backdrop, things, the_plot):
  self.n = np.random.randint(0, 3, dtype=np.int32)     # REFUSED


def _p(self, actions, board, layers, backdrop, things, the_plot):
  self.n = np.random.choice(3, p=None)                 # REFUSED


def _replace(self, actions, board, layers, backdrop, things, the_plot):
  self.n = np.random.choice(3, replace=True)           # REFUSED


def _step(self, actions, board, layers, backdrop, things, the_plot):
  self.n = random.randrange(0, 10, 2)                  # REFUSED


def _float_in_variable(self, actions, board, layers, backdrop, things, the_plot):
  x = np.random.rand()                                 # REFUSED
  del x


def _float_arithmetic(self, actions, board, layers, backdrop, things, the_plot):
  self.n = int(random.random() * 10)                   # REFUSED


def _float_against_a_register(self, actions, board, layers, backdrop, things, the_plot):
  if np.random.rand() < self.n:                        # REFUSED
    pass


def _chained_float(self, actions, board, layers, backdrop, things, the_plot):
  if 0.1 < np.random.rand() < 0.5:                     # REFUSED
    pass


def _non_literal_choice(self, actions, board, layers, backdrop, things, the_plot):
  self.n = np.random.choice(SEQ)                       # REFUSED


def _python_choice_of_a_number(self, actions, board, layers, backdrop, things, the_plot):
  self.n = random.choice(self.n)                       # REFUSED


def _empty_literal_choice(self, actions, board, layers, backdrop, things, the_plot):
  self.n = random.choice(())                           # REFUSED


def _private_generator(self, actions, board, layers, backdrop, things, the_plot):
  self.n = np.random.RandomState(3).randint(4)         # REFUSED


def _default_rng(self, actions, board, layers, backdrop, things, the_plot):
  self.n = np.random.default_rng().integers(4)         # REFUSED


def _generator_attribute(self, actions, board, layers, backdrop, things, the_plot):
  self.n = self.rng.randint(4)                         # REFUSED


def _uniform(self, actions, board, layers, backdrop, things, the_plot):
  if random.uniform(0, 1) < 0.5:                       # REFUSED
    pass


REFUSED = [(_size, 'the call np.random.randint()'), (_dtype, 'the call np.random.randint()'),
           (_p, 'the call np.random.choice()'), (_replace, 'the call np.random.choice()'),
           (_step, 'the call random.randrange()'),
           (_float_in_variable, 'the call np.random.rand()'),
           (_float_arithmetic, 'the call random.random()'),
           (_float_against_a_register, 'the call np.random.rand()'),
           (_chained_float, 'the call np.random.rand()'),
           (_non_literal_choice, 'the call np.random.choice()'),
           (_python_choice_of_a_number, 'the call random.choice()'),
           (_empty_literal_choice, 'the call random.choice()'),
           (_private_generator, 'the call np.random.RandomState(3).randint()'),
           (_default_rng, 'the call np.random.default_rng()'),
           (_generator_attribute, 'the call self.rng.randint()'),
           (_uniform, 'the call random.uniform()')]


@pytest.mark.parametrize('update,what', REFUSED, ids=[u.__name__ for u, _ in REFUSED])
def test_refused_draw_names_class_line_and_construct(update, what):
  msg = rg.assert_refused(rg.walker(update), what)
  assert '# REFUSED' in msg, msg


def test_games_without_draws_lower_with_no_streams():
  mod = rg.load('compiled_games.py')
  compiler.register(*mod.CLASSES)
  try:
    for make in mod.GAMES.values():
      lowered = lowering.lower(make(0))
      assert lowered.rng_streams == () and lowered.program_arg[1] == 0
      assert not lowered.needs_rng
  finally:
    compiler.unregister(*mod.CLASSES)


# ------------------------------------------------------- the draw restatement --

_EDGES = [(0, 1), (0, 2), (0, 3), (-7, -2), (-3, -2), (0, 2 ** 16), (0, 2 ** 16 + 1),
          (-2 ** 30, 1), (0, 2 ** 30 + 1), (-2 ** 31, 0), (-2 ** 31, 1), (-2 ** 31, 2 ** 31 - 1),
          (2 ** 31 - 2, 2 ** 31 - 1), (5, 5), (5, 4)]


def _numpy_words(rs):
  _, key, pos = rs.get_state()[:3]
  return [int(w) for w in key] + [int(pos)]


@pytest.mark.parametrize('seed', [0, 1, 12345])
def test_numpy_restatement_matches_random_state(seed):
  rs = np.random.RandomState(seed)
  words = _numpy_words(rs)
  for rep in range(60):                     # well past one twist (624 outputs)
    for low, high in _EDGES:
      want = None
      try:
        want = int(rs.randint(low, high))
      except ValueError:
        pass
      assert ocompiled.randint(words, _lib.RAND_NUMPY, low, high) == want, (seed, rep, low, high)
      assert words == _numpy_words(rs), (seed, rep, low, high)
    assert int(rs.choice(1)) == ocompiled.randint(words, _lib.RAND_NUMPY, 0, 1) == 0
    with pytest.raises(ValueError):
      rs.choice(0)
    assert ocompiled.randint(words, _lib.RAND_NUMPY, 0, 0) is None
    assert rs.choice((4, -1, 6)) == (4, -1, 6)[ocompiled.randint(words, _lib.RAND_NUMPY, 0, 3)]
    assert rs.random_sample() == ocompiled.random53(words)
    assert words == _numpy_words(rs)


@pytest.mark.parametrize('seed', [0, 1, 12345])
def test_python_restatement_matches_random(seed):
  r = random.Random(seed)
  words = list(r.getstate()[1])
  for rep in range(60):
    for low, high in _EDGES:
      want = None
      try:
        want = r.randrange(low, high)
      except ValueError:
        pass
      assert ocompiled.randint(words, _lib.RAND_PYTHON, low, high) == want, (seed, rep, low, high)
      assert words == list(r.getstate()[1]), (seed, rep, low, high)
      if high - 1 >= low:                   # randint(a, b) over [a, b]: up to 2^32 values
        assert r.randint(low, high) == ocompiled.randint(
            words, _lib.RAND_PYTHON_CLOSED, low, high), (seed, rep, low, high)
        assert words == list(r.getstate()[1])
    assert r.randint(-2 ** 31, 2 ** 31 - 1) == ocompiled.randint(
        words, _lib.RAND_PYTHON_CLOSED, -2 ** 31, 2 ** 31 - 1)
    assert r.randrange(1) == ocompiled.randint(words, _lib.RAND_PYTHON, 0, 1) == 0
    assert r.choice((4, -1, 6)) == (4, -1, 6)[ocompiled.randint(words, _lib.RAND_PYTHON, 0, 3)]
    assert r.random() == ocompiled.random53(words)
    assert words == list(r.getstate()[1])


# ------------------------------------------------------------ the C boundary --

def test_rng_slots_are_checked_at_the_boundary(games):
  lib = _lib.load()
  lowered = lowering.lower(games.make_edges(0))
  spec = lowered.make_spec(True)
  assert spec.program_arg[1] == 2
  h = C.c_void_p()
  for bad in (-1, 3):
    spec.program_arg[1] = bad
    assert lib.pcl_create(C.byref(spec), 4, -1, C.byref(h)) == _lib.ERR_INVALID, bad
  spec.program_arg[1] = 2
  assert lib.pcl_create(C.byref(spec), 4, -1, C.byref(h)) == _lib.OK
  try:
    state = boundary_sweep._full_state()
    state.d_rng = None
    assert lib.pcl_bind_state(h, C.byref(state)) == _lib.ERR_INVALID
    assert lib.pcl_bind_state(h, C.byref(boundary_sweep._full_state())) == _lib.OK
    code = lowered.code.copy()
    assert rg.bind(lib, h, code) == _lib.OK
    at = {name: [i for i in ocompiled.instructions(code, code[1], len(code))
                 if code[i] == _lib.OP[name]] for name in ('RANDINT', 'RANDCMP', 'PICK')}
    cases = []
    for i in at['RANDINT'][:1]:
      cases += [(i + 1, 2), (i + 1, -1), (i + 2, 3), (i + 2, -1)]    # slot, rule
    for i in at['RANDCMP'][:1]:
      cases += [(i + 1, 2), (i + 2, 6), (i + 2, -1)]                 # slot, comparison
    for i in at['PICK'][:1]:
      cases += [(i + 1, 0), (i + 1, 65), (i + 1, len(code))]         # value count
    assert len(cases) == 10
    for where, value in cases:
      bad = code.copy()
      bad[where] = value
      assert rg.bind(lib, h, bad) == _lib.ERR_INVALID, (where, value)
    assert rg.bind(lib, h, code) == _lib.OK
  finally:
    lib.pcl_destroy(h)
  # a game without draws may not hold a draw
  spec.program_arg[1] = 0
  assert lib.pcl_create(C.byref(spec), 4, -1, C.byref(h)) == _lib.OK
  try:
    assert lib.pcl_bind_state(h, C.byref(boundary_sweep._full_state())) == _lib.OK
    assert rg.bind(lib, h, lowered.code) == _lib.ERR_INVALID
  finally:
    lib.pcl_destroy(h)
