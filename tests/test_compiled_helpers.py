"""CPU tests of helper calls in compiled update() code: the game's own methods and module
functions, inlined by `pycolab_b200.compiler` into the words the interpreter already runs.

  - the oracle interpreter (oracle/compiled.py) latches PCL_ENV_ERR_ARITH where the reference
    raised ZeroDivisionError (tests/golden/helper_divzero.npz), after every frame before it;
  - virtual dispatch: subclasses overriding a helper get their own code, the others share;
  - role-only helpers without an early return link to the words of their pasted-in twin;
  - a helper's local slots are freed when its call ends;
  - each refused form names the helper, its line and the call site;
  - pcl_bind_code accepts the linked words, on handles that reach no device.
"""

import inspect

import numpy as np
import pytest

import golden_cases as gc
import registered_games as rg
from pycolab_b200 import _lib, compiler, lowering
from pycolab_b200 import things as b_things
from pycolab_b200.errors import NotLoweredError
from pycolab_b200.prefab_parts import sprites as b_sprites


@pytest.fixture(scope='module')
def games():
  yield from rg.registered('helper_games.py')


def test_oracle_latches_arith_where_the_reference_divided_by_zero(games):
  """helper_divzero on the oracle: every frame before the reference's ZeroDivisionError,
  then PCL_ENV_ERR_ARITH (a case of test_registered_goldens too)."""
  rg.assert_oracle_replays(games, 'helper_divzero')


# ------------------------------------------------------------ virtual dispatch --

def test_overriding_subclasses_get_their_own_code(games):
  base, up, down = (compiler.registered(k) for k in (games.Bolt, games.UpBolt, games.DownBolt))
  assert len({id(base), id(up), id(down)}) == 3
  assert up.klass is down.klass is games.Bolt                 # the registered class
  assert up.methods['_fly'] is vars(games.UpBolt)['_fly']
  assert compiler.registered(games.StrayBolt) is base       # overrides nothing
  assert compiler.registered(games.DownBolt) is down        # compiled once

  class Again(games.UpBolt):
    pass
  assert compiler.registered(Again) is up                   # the helpers resolve as UpBolt's

  lowered = lowering.lower(games.make_bolts(0))
  entry = {ch: lowered.code[1 + i] for i, ch in enumerate(lowered.sprite_chars +
                                                         lowered.drape_chars)}
  assert entry[':'] == entry[';']                           # one class
  assert len({entry['!'], entry[':'], entry['^'], entry['P'], entry['X']}) == 5
  assert any(ins[0] == 'RANDINT' for ins in down.ir)
  assert not any(ins[0] == 'RANDINT' for ins in up.ir + base.ir)


def test_subclass_compilations_do_not_keep_their_classes_alive(games):
  import gc
  import weakref

  def _fly(self, board, layers, things, the_plot):
    self._south(board, the_plot)
  made = type('Made', (games.Bolt,), {'_fly': _fly, '__module__': games.Bolt.__module__})
  comp = compiler.registered(made)
  assert comp is not compiler.registered(games.Bolt) and comp is compiler.registered(made)
  gone = weakref.ref(made)
  del made
  gc.collect()
  assert gone() is None
  assert ('MOVE', 4) in comp.ir


def _walks_north(self, actions, board, layers, backdrop, things, the_plot):
  if actions == 0:
    self._north(board, the_plot)
  self.n = 1 if self._north(board, the_plot) is None else 0


def _north_is_south(self, board, the_plot):
  return self._south(board, the_plot)


def test_an_override_of_a_motion_helper_runs_as_python_would():
  base = _case(_walks_north)
  sub = type('Sub', (base,), {'_north': _north_is_south, '__module__': __name__})
  compiler.register(base)
  try:
    assert compiler.registered(base).methods['_north'] is b_sprites.MazeWalker._north
    comp = compiler.registered(sub)
    assert comp is not compiler.registered(base)
    moves = [ins for ins in comp.ir if ins[0] == 'MOVE']
    assert moves == [('MOVE', 4), ('MOVE', 4)]
    assert moves == [ins for ins in compiler.compile_class(sub).ir if ins[0] == 'MOVE']
    assert compiler.registered(type('Plain', (base,), {})) is compiler.registered(base)
  finally:
    compiler.unregister(base)


def test_a_new_registration_drops_the_subclass_compilations(games):
  up = compiler.registered(games.UpBolt)
  compiler.register(games.Bolt)
  assert compiler.registered(games.UpBolt) is not up
  assert compiler.registered(games.UpBolt).ir == up.ir


# ------------------------------------------------------------ inlining --

def _case(update, base=b_sprites.MazeWalker, **helpers):
  helpers.update(update=update, __module__=__name__)
  return type('Case', (base,), helpers)


def _link(klass, keys=()):
  return compiler.link({'P': compiler.compile_class(klass)}, 'P', '', 7, 9, list(keys)).tolist()


def _with_helpers(self, actions, board, layers, backdrop, things, the_plot):
  self._steer(actions, board, the_plot)
  if self.visible:
    self._count(the_plot, things)


def _steer(self, act, board, the_plot):
  if act == 0:
    self._north(board, the_plot)
  elif act == 1:
    self._south(board, the_plot)
  else:
    self._stay(board, the_plot)


def _count(self, plot, all_things):
  plot['n'] += 1
  if all_things['P'].position.row == 2:
    plot.add_reward(1)


def _pasted(self, actions, board, layers, backdrop, things, the_plot):
  if actions == 0:
    self._north(board, the_plot)
  elif actions == 1:
    self._south(board, the_plot)
  else:
    self._stay(board, the_plot)
  if self.visible:
    the_plot['n'] += 1
    if things['P'].position.row == 2:
      the_plot.add_reward(1)


def test_role_only_helpers_link_to_the_words_of_their_pasted_twin():
  helpers = _case(_with_helpers, _steer=_steer, _count=_count)
  assert _link(helpers, ['n']) == _link(_case(_pasted), ['n'])


def _early(self, actions, board, layers, backdrop, things, the_plot):
  self.n = self._pick(actions) + _twice(self.n)
  if self._pick(actions) == 2:
    self._north(board, the_plot)


def _pick(self, act):
  if act == 0:
    return 1
  elif act == 1:
    return 2
  return 3


def _twice(x, by=2):
  return x * by


def test_value_returns_jump_forward_to_the_helpers_end():
  ir = compiler.compile_class(_case(_early, _pick=_pick)).ir
  jumps = [ins for ins in ir if ins[0] in ('JMP', 'JZ', 'JNZ')]
  assert ('MUL',) in ir and ir.count(('PUSH', 2)) >= 3
  assert all(ins[1][0] == 'label' for ins in jumps)
  # every label is placed after each jump to it
  at = {ins[1]: i for i, ins in enumerate(ir) if ins[0] == 'LABEL'}
  assert all(at[ins[1][1]] > i for i, ins in enumerate(ir) if ins[0] in ('JMP', 'JZ', 'JNZ'))


def _nine(self):
  a, b = self.position
  c, d = self.position
  e, f = self.position
  g, h = self.position
  i = a + b + c + d + e + f + g + h
  self.total = i


def _sequential(self, actions, board, layers, backdrop, things, the_plot):
  x = 1
  self._nine()
  self._nine()
  y = x + 1
  self.total = y


def _seventeen(self, actions, board, layers, backdrop, things, the_plot):
  self._nine()
  a, b = self.position
  c, d = self.position
  e, f = self.position
  g, h = self.position
  self.total = a + b + c + d + e + f + g + h


def _inside(self, actions, board, layers, backdrop, things, the_plot):
  x = 1
  self._nine_of(x)
  self.total = x


def _nine_of(self, x):
  self._nine()


def test_sequential_calls_reuse_local_slots():
  ir = compiler.compile_class(_case(_sequential, _nine=_nine)).ir
  stores = [ins[1] for ins in ir if ins[0] == 'STORE']
  assert max(stores) == 9                     # x in 0, the helper's nine in 1-9, twice
  assert stores.count(9) == 2 and stores[-1] == 1   # y reuses the helper's first slot
  compiler.compile_class(_case(_seventeen, _nine=_nine))      # 9 freed, then 8
  ir = compiler.compile_class(_case(_inside, _nine=_nine, _nine_of=_nine_of)).ir
  assert max(ins[1] for ins in ir if ins[0] == 'STORE') == 10  # x, the argument x, then nine


def _seventeen_live(self, actions, board, layers, backdrop, things, the_plot):
  a, b = self.position
  c, d = self.position
  e, f = self.position
  g, h = self.position
  self._nine()                                          # CALL


def test_live_slots_over_the_limit_are_refused():
  with pytest.raises(NotLoweredError, match='more than 16 local slots') as e:
    compiler.compile_class(_case(_seventeen_live, _nine=_nine))
  assert '_nine, line' in str(e.value) and 'called from Case.update' in str(e.value)


def _mark_char(self, board, ch, the_plot, reward=1):
  if chr(board[1, 1]) == ch:
    the_plot.add_reward(reward)


def _char_marks(self, actions, board, layers, backdrop, things, the_plot):
  self._mark(board, 'P', the_plot)
  self._mark(board, '#', the_plot, reward=2)


def test_a_character_argument_specialises_the_body():
  ir = compiler.compile_class(_case(_char_marks, _mark=_mark_char)).ir
  assert ('PUSH', ord('P')) in ir and ('PUSH', ord('#')) in ir
  assert ir.count(('REWARD',)) == 2


# ------------------------------------------------------------ refusals --

def _calls_h(self, actions, board, layers, backdrop, things, the_plot):
  self._h(board, the_plot)                              # CALL


def _calls_h_value(self, actions, board, layers, backdrop, things, the_plot):
  self.n = self._h(1)                                   # CALL


def _h_varargs(self, *rest):
  pass


def _h_kwargs(self, board, **rest):
  pass


def _h_kwonly(self, board, *, the_plot=None):
  pass


def _h_static(board, the_plot):
  pass


def _h_generator(self, board, the_plot):
  yield 1


_h_lambda = lambda self, board, the_plot: None


def _closure():
  k = 1

  def _h_closure(self, board, the_plot):
    self.n = k
  return _h_closure


def _h_nested(self, board, the_plot):
  def inner():                                          # REFUSED
    pass


def _h_super(self, board, the_plot):
  super()._north(board, the_plot)                       # REFUSED


def _h_other(self, board, the_plot):
  things['P']._m()                                      # REFUSED


def _h_assign_role(self, board, the_plot):
  board = 1                                             # REFUSED


def _h_for(self, board, the_plot):
  for _ in range(2):                                    # REFUSED
    pass


def _h_log(self, board, the_plot):
  the_plot.log('hello')                                 # REFUSED


def _h_falls(self, x):
  if x:
    return 1


def _h_mixed(self, x):
  if x:
    return 1
  return self.position                                  # REFUSED


def _h_recursive(self, board, the_plot):
  self._h(board, the_plot)


def _h_a(self, board, the_plot):
  self._b(board, the_plot)


def _h_b(self, board, the_plot):
  self._h(board, the_plot)


def _decorate(fn):
  return fn


@_decorate
def _h_decorated(self, board, the_plot):
  pass


_ns = {'__name__': __name__}
exec('def _h_no_source(self, board, the_plot):\n  pass\n', _ns)


def _def_line(fn):
  return fn.__code__.co_firstlineno


def _marked(fn):
  lines, first = inspect.getsourcelines(fn)
  return first + [i for i, l in enumerate(lines) if '# REFUSED' in l][0]


# (helper, how it is attached, what, its line, the update that calls it)
HELPER_REFUSED = [
    (_h_varargs, None, '*args, **kwargs or a keyword-only parameter', None, _calls_h),
    (_h_kwargs, None, '*args, **kwargs or a keyword-only parameter', None, _calls_h),
    (_h_kwonly, None, '*args, **kwargs or a keyword-only parameter', None, _calls_h),
    (_h_static, staticmethod, 'a staticmethod helper', None, _calls_h),
    (_h_static, classmethod, 'a classmethod helper', None, _calls_h),
    (_h_static, property, 'a property helper', None, _calls_h),
    (_h_generator, None, 'a generator', None, _calls_h),
    (_h_lambda, None, 'a lambda', None, _calls_h),
    (_closure(), None, 'a closure over k', None, _calls_h),
    (_h_decorated, None, 'a decorated helper', None, _calls_h),
    (_ns['_h_no_source'], None, 'a helper whose source is not available', None, _calls_h),
    (_h_nested, None, 'FunctionDef', _marked, _calls_h),
    (_h_super, None, 'the call super()._north()', _marked, _calls_h),
    (_h_other, None, "the call things['P']._m()", _marked, _calls_h),
    (_h_assign_role, None, 'assigning an update() argument', _marked, _calls_h),
    (_h_for, None, 'For', _marked, _calls_h),
    (_h_log, None, 'the call the_plot.log()', _marked, _calls_h),
    (_h_falls, None, 'a helper that returns a number and can fall off its end', None,
     _calls_h_value),
    (_h_mixed, None, 'returning a number and a position', _marked, _calls_h_value),
    (_h_recursive, None, 'recursion (_h_recursive -> _h_recursive)', None, _calls_h),
]


@pytest.mark.parametrize('helper,wrap,what,line,update', HELPER_REFUSED,
                         ids=['{}-{}'.format(h.__name__, getattr(w, '__name__', 'plain'))
                              for h, w, _, _, _ in HELPER_REFUSED])
def test_refused_helper_names_itself_its_line_and_the_call_site(helper, wrap, what, line, update):
  at = (line or _def_line)(helper)
  call = _marked_call(update)
  with pytest.raises(NotLoweredError) as e:
    compiler.compile_class(_case(update, _h=wrap(helper) if wrap else helper))
  msg = str(e.value)
  assert '{}.{}, line {}: '.format(__name__, helper.__qualname__, at) in msg, msg
  assert what in msg, msg
  assert msg.endswith('called from Case.update, line {})'.format(call)), msg


def _marked_call(update):
  lines, first = inspect.getsourcelines(update)
  return first + [i for i, l in enumerate(lines) if '# CALL' in l][0]


def test_mutual_recursion_names_the_cycle():
  with pytest.raises(NotLoweredError) as e:
    compiler.compile_class(_case(_calls_h, _h=_h_a, _b=_h_b))
  msg = str(e.value)
  assert 'recursion (_h_a -> _h_b -> _h_a)' in msg, msg
  assert '(called from _h_b, line {}, called from _h_a, line {}, called from Case.update'.format(
      _def_line(_h_b) + 1, _def_line(_h_a) + 1) in msg, msg


def _d0(x):
  return _d1(x)


def _d1(x):
  return _d2(x)


def _d2(x):
  return _d3(x)


def _d3(x):
  return _d4(x)


def _d4(x):
  return _d5(x)


def _d5(x):
  return _d6(x)


def _d6(x):
  return _d7(x)


def _d7(x):
  return _d8(x)


def _d8(x):
  return x + 1


def _calls_deep(self, actions, board, layers, backdrop, things, the_plot):
  self.n = _d0(1)


def _calls_eight(self, actions, board, layers, backdrop, things, the_plot):
  self.n = _d1(1)


def test_helpers_nest_eight_deep():
  compiler.compile_class(_case(_calls_eight))
  with pytest.raises(NotLoweredError, match='_d8, line .*: helpers nested more than 8 deep'):
    compiler.compile_class(_case(_calls_deep))


def _passes_curtain(self, actions, board, layers, backdrop, things, the_plot):
  self._h(self.curtain)


def _passes_char(self, actions, board, layers, backdrop, things, the_plot):
  self._h(chr(board[1, 1]))


def _passes_self(self, actions, board, layers, backdrop, things, the_plot):
  self.n = _twice(self)


def _h_one(self, x):
  pass


@pytest.mark.parametrize('update,what', [
    (_passes_curtain, 'the argument x=self.curtain of self._h()'),
    (_passes_char, 'the argument x=chr(board[1, 1]) of self._h()'),
    (_passes_self, 'the argument x=self of _twice()')])
def test_refused_arguments_are_named(update, what):
  with pytest.raises(NotLoweredError) as e:
    compiler.compile_class(_case(update, base=b_things.Drape, _h=_h_one))
  assert 'Case.update, line' in str(e.value) and what in str(e.value), str(e.value)


def _void_into_local(self, actions, board, layers, backdrop, things, the_plot):
  x = self._h(board, the_plot)                          # CALL


def _void_into_register(self, actions, board, layers, backdrop, things, the_plot):
  self.n = self._h(board, the_plot)                     # CALL


def _void_as_truth(self, actions, board, layers, backdrop, things, the_plot):
  if self._h(board, the_plot):                          # CALL
    pass


def _void_in_arithmetic(self, actions, board, layers, backdrop, things, the_plot):
  self.n = 1 + self._h(board, the_plot)                 # CALL


@pytest.mark.parametrize('update', [_void_into_local, _void_into_register, _void_as_truth,
                                    _void_in_arithmetic])
def test_the_value_of_a_helper_that_returns_nothing_is_refused(update):
  with pytest.raises(NotLoweredError) as e:
    compiler.compile_class(_case(update, _h=_steer_north))
  msg = str(e.value)
  assert 'Case.update, line {}: the value of self._h(), which returns nothing'.format(
      _marked_call(update)) in msg, msg


def _h_positional_only(self, x, /):
  self.n = x


def _keyword_to_positional_only(self, actions, board, layers, backdrop, things, the_plot):
  self._h(x=1)                                          # CALL


def _positional_to_positional_only(self, actions, board, layers, backdrop, things, the_plot):
  self._h(1)


def test_a_positional_only_parameter_takes_no_keyword():
  with pytest.raises(NotLoweredError, match=r'these arguments of self._h\(\)'):
    compiler.compile_class(_case(_keyword_to_positional_only, _h=_h_positional_only))
  compiler.compile_class(_case(_positional_to_positional_only, _h=_h_positional_only))


def _stdlib_named(x):
  return x + 1


_stdlib_named.__module__ = 'code'             # a game module named like a standard one


def _calls_stdlib_named(self, actions, board, layers, backdrop, things, the_plot):
  self.n = _stdlib_named(1)


def _calls_stdlib(self, actions, board, layers, backdrop, things, the_plot):
  self.n = inspect.cleandoc(1)


def _calls_numpy(self, actions, board, layers, backdrop, things, the_plot):
  self.n = np.roll(1, 1)


def test_the_games_code_is_told_by_its_file():
  ir = compiler.compile_class(_case(_calls_stdlib_named)).ir
  assert ('ADD',) in ir
  with pytest.raises(NotLoweredError, match=r'the call inspect.cleandoc\(\) is not compiled'):
    compiler.compile_class(_case(_calls_stdlib))
  with pytest.raises(NotLoweredError, match=r'the call np.roll\(\) is not compiled'):
    compiler.compile_class(_case(_calls_numpy))


def _unknown_method(self, actions, board, layers, backdrop, things, the_plot):
  self._fly(board, the_plot)


def test_calls_that_resolve_to_no_user_helper_keep_their_refusal():
  with pytest.raises(NotLoweredError, match=r'the call self._fly\(\) is not compiled'):
    compiler.compile_class(_case(_unknown_method))
  with pytest.raises(NotLoweredError, match=r'_north in a plain class'):
    compiler.compile_class(_case(_calls_h, base=b_things.Sprite, _h=_steer_north))


def _steer_north(self, board, the_plot):
  self._north(board, the_plot)


# ------------------------------------------------------------ pcl_bind_code --

@pytest.mark.parametrize('game,level', [('bolts', 0), ('bolts', 1), ('chaser', 0),
                                        ('chaser', 1), ('divzero', 0)])
def test_bind_code_accepts_inlined_helpers(games, game, level):
  lib = _lib.load()
  lowered = lowering.lower(games.GAMES[game](level))
  h = rg.handle(lib, lowered.make_spec(True))
  try:
    assert rg.bind(lib, h, lowered.code) == _lib.OK
  finally:
    lib.pcl_destroy(h)
