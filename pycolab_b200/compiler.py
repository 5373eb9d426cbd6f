"""Compile entity classes' own `update()` methods to device bytecode (`PCL_PROG_COMPILED`).

    from pycolab_b200 import compiler
    compiler.register(my_game.PlayerSprite, my_game.CoinDrape)

`register` opts classes in: their `update()` source (`inspect.getsource` + `ast`) is
compiled to the stack bytecode of include/pcl.h (`PCL_OP_*`), and from then on
`lowering.lower` runs games made of registered classes on the compiled step program
(csrc/compiled.cu) instead of refusing them.  Classes that are not registered behave
as before.

The subset (everything else raises `NotLoweredError` naming the class, the source line
and the construct):
  entities    MazeWalker subclasses (any impassable set, confined or not, egocentric or
              not), plain Sprite subclasses (things.Sprite, not MazeWalker), Scrolly
              subclasses and plain Drape subclasses, all in one scrolling group; the
              Scrollys' patterns all of one shape; a Backdrop subclass with its own
              update(self, actions, board, layers, things, the_plot), which has no
              registers and runs before update group 0;
  statements  if / elif / else, return, pass; `del` and docstrings compile to nothing;
              local variables holding an int, a bool, a position or a motion result;
              `r, c = <position>`;
              `self.<attr>` and `the_plot['key']` with =, +=, -=, *=, //=, %=;
              motion helpers (`self._north(board, the_plot)` ... `self._stay(...)`; on
              Scrollys `self._north(the_plot)` ...), also as
              `(self._east if c else self._west)(...)`,
              `self._teleport(pos)`, `the_plot.add_reward(x)`,
              `the_plot.terminate_episode([discount])`, `the_plot.change_default_discount(c)`;
              on plain drapes `self.curtain[cell] = v` and `self.curtain[:] = v`;
              on plain Sprites `self._position = <position>` (not a bare tuple: upstream
              `.row` would fail on it later) and `self._visible = <truth value>`;
              on Scrollys `self.whole_pattern[cell] = v` (their own pattern only);
              on a Backdrop `self.curtain[cell] = v`, `self.curtain[:] = v` and
              `self.curtain[a:b, :] = np.roll(self.curtain[a:b, :], shift, axis)` (also
              `[a:b]`, or the whole curtain; int literal bounds, the same band on both
              sides, the literal axis 0 or 1, np.roll found as draws are), where v is a
              palette look-up, ord('c'), an int literal 0..255, a board or curtain cell,
              a bool, or `x if c else y` of these (each lies in 0..255);
  values      `actions` (==, !=, in, is None only), int and bool literals (float literals
              only as a reward or a discount), + - * // % and unary -, comparisons
              (chained, position against position or tuple), `in` over a literal
              tuple / list / string, and / or / not, `x if c else y`, `is None` on
              motion results, int(), ord('c'), chr(cell) against characters, positions
              (`.position`, `.virtual_position`, `.corner`, `.row`, `.col`, [0], [1]),
              `.visible`, `self._position` / `self._visible` of a plain Sprite,
              `self.Position(r, c)` / `Position(row=r, col=c)` (also as `Sprite.Position`
              through update()'s module globals, e.g. `things.Sprite.Position`),
              `the_plot.frame`, `the_plot['key']`, `the_plot.get('key')`,
              `board[cell]`, `backdrop.curtain[cell]`, `layers['X'][cell]`,
              `self.curtain[cell]`, `things['X'].position / .visible / .curtain[cell]`,
              `.curtain.any()` (a Scrolly's curtain is its pattern window);
              `board.shape`, `board.shape[0]`, `board.shape[1]`; in a Backdrop also
              `self.curtain.shape`, `self.curtain[cell]` (its live curtain) and
              `self.palette.X` / `self.palette['X']` (aliases included; lowering checks
              the character against the game's palette);
              of Scrollys (`self` or `things['X']`): `.pattern_position_prescroll(pos,
              the_plot)`, `.pattern_position_postscroll(pos, the_plot)`,
              `.whole_pattern[cell]`, `.whole_pattern.any()`.
  draws       from the global generators, whose functions are found through update()'s
              module globals and compared by identity (so `import numpy as np`,
              `from numpy import random as npr` and `from random import randint` all
              work), with int operands and no keywords:
                NumPy's RandomState: `np.random.randint(high)`, `randint(low, high)`,
                `choice(n)`, `choice(<literal tuple / list of ints>)`;
                Python's Random: `random.randint(a, b)`, `randrange(stop)`,
                `randrange(start, stop)`, `choice(<literal tuple / list of ints>)`;
                a float draw, `np.random.rand()` / `random()` / `random_sample()` or
                `random.random()`, only as one side of a comparison with a number literal.
              Each draw continues the env's copy of that generator on the device
              (include/pcl.h PCL_OP_RANDINT) and yields what the generator would.
  helpers     calls of the game's own code, inlined where they stand (there is no call
              opcode, so every jump stays forward and a helper costs nothing at run time):
              `self.name(...)` where `name` resolves along the entity class's MRO to a plain
              function of the game's code (methods of this package's classes keep the
              treatment above; a game's override of one, `_north` say, is inlined as Python
              would call it), and `name(...)` of a plain function of the game's code, found
              through the module globals as draws are.  The game's code is every function
              but this package's, NumPy's and the standard library's.  Arguments are positional or keyword,
              defaults int / bool / None / one-character string literals.  An update()
              argument (board, layers, things, backdrop, the_plot, actions) passed under any
              parameter name stands for it inside the helper; a one-character string literal
              is a constant of the body, specialised per call site (`things[ch]`,
              `layers[ch]`, `board[p] == ch`); any other argument is an int, bool, position or
              motion result, evaluated once, left to right, into fresh local slots that are
              freed when the call ends (PCL_CODE_LOCALS bounds the deepest chain of live
              slots).  A helper returns nothing (`return`, `return None`, `return <call
              returning nothing>` such as `return self._teleport(p)`), or a value of one type
              on every path: a number or a position, which may not fall off the end, or a
              motion result, which falls off as None.  A value used as a statement is
              discarded.  Helpers nest up to MAX_HELPER_DEPTH deep; recursion, `*args`,
              `**kwargs`, keyword-only parameters, decorators (staticmethod, classmethod,
              property), lambdas, closures, generators, `super()` and another entity's methods
              are refused, naming the helper, its line and each call site.  Inside a helper
              `self.<attr>`, Plot keys, draws and entity look-ups are update()'s.  When a
              subclass overrides a helper, `registered` compiles update() for it again.
Int and bool attributes of `self` become per-entity registers and `the_plot` keys plot
registers; their values are read from the live objects when the game is lowered.  An
attribute used as a position (`self._start = self.position`, `self._position =
self._start`, `board[self._start]`) is a position attribute and takes two registers; its
first use in update() fixes which it is, and a later use as the other is refused.  A walker
and a Scrolly have 3 registers, an egocentric walker 1, a plain Sprite 5, a plain drape 8,
the plot 4.  Integers are 32 bits on the device; values outside int32 wrap.  After a facade
step a register is written back with the type (bool, int, Position or tuple) its value had
at lowering.
"""

import ast
import inspect
import os
import random
import struct
import sysconfig
import textwrap
import types
import weakref

import numpy as np

from pycolab_b200 import _lib
from pycolab_b200 import engine as engine_lib
from pycolab_b200 import things
from pycolab_b200.errors import NotLoweredError
from pycolab_b200.prefab_parts import drapes as prefab_drapes
from pycolab_b200.prefab_parts import sprites as prefab_sprites

_REGISTRY = {}                # class -> Compiled
_VARIANTS = {}                # registered class -> {subclass: its Compiled}, weak in the subclass

_PARAMS = ('self', 'actions', 'board', 'layers', 'backdrop', 'things', 'the_plot')
_BACKDROP_PARAMS = ('self', 'actions', 'board', 'layers', 'things', 'the_plot')
_MOTIONS = {'_north': 0, '_northeast': 1, '_east': 2, '_southeast': 3, '_south': 4,
            '_southwest': 5, '_west': 6, '_northwest': 7, '_stay': 8}
_BINOPS = {ast.Add: 'ADD', ast.Sub: 'SUB', ast.Mult: 'MUL', ast.FloorDiv: 'FLOORDIV',
           ast.Mod: 'MOD'}
_CMPOPS = {ast.Eq: 'EQ', ast.NotEq: 'NE', ast.Lt: 'LT', ast.LtE: 'LE', ast.Gt: 'GT',
           ast.GtE: 'GE'}
_POSITIONS = {'position': (_lib.FIELD_ROW, _lib.FIELD_COL),
              'virtual_position': (_lib.FIELD_VROW, _lib.FIELD_VCOL)}
# Registers per entity: sprite record AUX0-AUX2, a Scrolly's AUX0-AUX2, every word of a plain
# drape's record.  An egocentric walker keeps its permits in AUX0 / AUX1: it has AUX2 only.
# A plain Sprite has no virtual position: its registers are VROW, VCOL and AUX0-AUX2.
MAX_REGISTERS = {'sprite': 3, 'plain': 5, 'scrolly': 3, 'drape': _lib.DRAPE_WORDS}
MAX_EGOCENTRIC_REGISTERS = 1
_PATTERN_POSITIONS = {'pattern_position_prescroll': 'PRESCROLL',
                      'pattern_position_postscroll': 'POSTSCROLL'}
MAX_PLOT_KEYS = 4
# The generator functions a draw may call: (function, stream, kind).
_DRAWS = ((np.random.randint, 'numpy', 'randint'), (np.random.choice, 'numpy', 'choice'),
          (np.random.rand, 'numpy', 'float'), (np.random.random, 'numpy', 'float'),
          (np.random.random_sample, 'numpy', 'float'),
          (random.randint, 'python', 'randint'), (random.randrange, 'python', 'randrange'),
          (random.choice, 'python', 'choice'), (random.random, 'python', 'float'))
# `x op draw` as `draw op' x`.
_FLIPPED = {ast.Eq: ast.Eq, ast.NotEq: ast.NotEq, ast.Lt: ast.Gt, ast.LtE: ast.GtE,
            ast.Gt: ast.Lt, ast.GtE: ast.LtE}
_TYPE_NAMES = {'int': 'number', 'pos': 'position', 'motion': 'motion result', 'char': 'character'}
# Stack words of the values a helper takes or returns.
_WIDTH = {'int': 1, 'motion': 1, 'pos': 2}
# update() arguments a helper may take, under any parameter name.
_ROLES = ('actions', 'board', 'layers', 'backdrop', 'things', 'the_plot')
# What the compiler keeps of the function whose body it compiles, saved around an inlined helper.
_FRAME = ('lines', 'first', 'globals', 'role', 'locals', 'where', 'short', 'ret')
MAX_HELPER_DEPTH = 8
# A plain Sprite's own state (things.py:339-391), read and written in place.
_SPRITE_STATE = ('_position', '_visible')


def _f32_bits(x):
  return struct.unpack('<i', struct.pack('<f', float(x)))[0]


def _f64_halves(x):
  lo, hi = struct.unpack('<ii', struct.pack('<d', float(x)))
  return lo, hi


class Compiled(object):
  """One class's update(), compiled with symbolic operands (`link` resolves them):
  ('attr', name) a register, ('key', name) a plot key, ('ent', char) an entity,
  ('label', n) a code address, ('rows',) / ('cols',) the board shape, ('rng', stream) the
  RNG slot of a generator."""

  def __init__(self, klass, kind, ir, attrs, keys, float_reward, streams=(), attr_types=None,
               methods=None):
    self.klass, self.kind, self.ir = klass, kind, ir
    self.attrs = attrs            # register names, in slot order
    # 'int' (ints and bools, one register) or 'pos' (a position, two: row, then col)
    self.attr_types = dict(attr_types or {})
    self.keys = keys              # the_plot keys it reads or writes
    self.float_reward = float_reward
    self.streams = list(streams)  # generators it draws from ('numpy', 'python'), first use first
    # name -> the class attribute each inlined `self.name(...)` resolved to on `klass`
    self.methods = dict(methods or {})

  def width(self, name):
    return 2 if self.attr_types.get(name) == 'pos' else 1

  def slot(self, name):
    """The first register of attribute `name`."""
    return sum(self.width(a) for a in self.attrs[:self.attrs.index(name)])

  @property
  def n_registers(self):
    return sum(self.width(a) for a in self.attrs)


def register(*classes):
  """Compile each class's update() and make `lowering` run it on the device.
  Returns its argument (so `@compiler.register` decorates a class)."""
  for klass in classes:
    _REGISTRY[klass] = compile_class(klass)
    _VARIANTS.pop(klass, None)
  return classes[0] if len(classes) == 1 else classes


def unregister(*classes):
  for klass in classes:
    _REGISTRY.pop(klass, None)
    _VARIANTS.pop(klass, None)


def registered(cls):
  """The `Compiled` of the registered class along `cls`'s MRO whose update() `cls` uses,
  or None.  When a method that update() calls as `self.name(...)` resolves differently on
  `cls` (a subclass overrides a helper or a motion helper), this is a compilation for `cls`,
  shared with every class whose methods resolve as `cls`'s do.  Its `klass` is the
  registered class, and the cache holds subclasses weakly, so classes made at run time
  can be freed."""
  for klass in cls.__mro__:
    if klass in _REGISTRY:
      if cls.update is not klass.update:
        return None
      variants = _VARIANTS.setdefault(klass, weakref.WeakKeyDictionary())
      if cls not in variants:
        for comp in [_REGISTRY[klass]] + list(variants.values()):
          if all(inspect.getattr_static(cls, name, None) is obj
                 for name, obj in comp.methods.items()):
            break
        else:
          comp = compile_class(cls)
          comp.klass = klass
        variants[cls] = comp
      return variants[cls]
  return None


def compile_class(klass):
  if not isinstance(klass, type):
    raise TypeError('register() takes classes, got {!r}'.format(klass))
  if issubclass(klass, prefab_sprites.MazeWalker):
    kind = 'sprite'
  elif issubclass(klass, things.Sprite):
    kind = 'plain'
  elif issubclass(klass, prefab_drapes.Scrolly):
    kind = 'scrolly'
  elif issubclass(klass, things.Drape):
    kind = 'drape'
  elif issubclass(klass, things.Backdrop):
    kind = 'backdrop'
  else:
    raise NotLoweredError('{}: only Sprite, MazeWalker, Scrolly, plain Drape and Backdrop '
                          'subclasses are compiled'.format(_name(klass)))
  if klass.update in (prefab_sprites.MazeWalker.update, things.Sprite.update,
                      things.Drape.update, things.Backdrop.update):
    raise NotLoweredError('{}: has no update() of its own to compile'.format(_name(klass)))
  return _Compiler(klass, kind).run()


def _name(klass):
  return '{}.{}'.format(klass.__module__, klass.__qualname__)


class _Compiler(object):

  def __init__(self, klass, kind):
    self.klass, self.kind = klass, kind
    fn = klass.update
    try:
      lines, self.first = inspect.getsourcelines(fn)
    except (OSError, TypeError):
      raise NotLoweredError('{}: the source of update() is not available'.format(_name(klass)))
    self.lines = lines
    self.globals = getattr(fn, '__globals__', {})
    tree = ast.parse(textwrap.dedent(''.join(lines)))
    self.fdef = tree.body[0]
    args = self.fdef.args
    params = _BACKDROP_PARAMS if kind == 'backdrop' else _PARAMS
    if (not isinstance(self.fdef, ast.FunctionDef) or len(args.args) != len(params) or
        args.vararg or args.kwarg or args.kwonlyargs or self.fdef.decorator_list):
      raise NotLoweredError('{}: update() must take the {} standard arguments'.format(
          _name(klass), 'six' if kind == 'backdrop' else 'seven'))
    self.role = {a.arg: role for a, role in zip(args.args, params)}
    self.ir = []
    self.n_labels = 0
    self.locals = {}              # name -> (first slot, type)
    self.n_slots = 0
    self.attrs, self.keys = [], []
    self.attr_types = {}
    self.float_reward = False
    self.streams = []
    # The function being compiled (update() or an inlined helper): see _FRAME.
    self.where = _name(klass) + '.update'
    self.short = klass.__qualname__ + '.update'
    self.ret = None               # an inlined helper's _Return, None in update()
    self.callers = []             # (short name, line) of each call site being inlined
    self.active = []              # the helpers being inlined, outermost first
    self.methods = {}             # name -> class attribute of each inlined self.name()
    self.helper_types = {}        # call node -> what the helper it inlines returns

  def run(self):
    self.stmts(self.fdef.body)
    self.emit('RET')
    return Compiled(self.klass, self.kind, self.ir, self.attrs, self.keys, self.float_reward,
                    self.streams, self.attr_types, self.methods)

  # -------------------------------------------------------------- helpers
  def refuse(self, node, what):
    line = self.first + getattr(node, 'lineno', 1) - 1
    text = self.lines[getattr(node, 'lineno', 1) - 1].strip()
    raise NotLoweredError('{}, line {}: {} is not compiled: {}{}'.format(
        self.where, line, what, text, self.called_from()))

  def called_from(self):
    """' (called from Case.update, line N)' inside an inlined helper, else ''."""
    if not self.callers:
      return ''
    return ' (called from {})'.format(', called from '.join(
        '{}, line {}'.format(name, line) for name, line in reversed(self.callers)))

  def emit(self, *ins):
    self.ir.append(ins)

  def label(self):
    self.n_labels += 1
    return ('label', self.n_labels)

  def place(self, lab):
    self.ir.append(('LABEL', lab[1]))

  def is_param(self, node, role):
    return isinstance(node, ast.Name) and self.role.get(node.id) == role

  def is_self(self, node):
    return self.is_param(node, 'self')

  def thing_char(self, node):
    """'X' of `things['X']`, else None."""
    if (isinstance(node, ast.Subscript) and self.is_param(node.value, 'things') and
        isinstance(node.slice, ast.Constant) and isinstance(node.slice.value, str)):
      return node.slice.value
    return None

  def plot_key(self, node):
    """'k' of `the_plot['k']`, else None."""
    if isinstance(node, ast.Subscript) and self.is_param(node.value, 'the_plot'):
      if isinstance(node.slice, ast.Constant) and isinstance(node.slice.value, str):
        return self.use_key(node.slice.value)
      self.refuse(node, 'a the_plot key that is not a string literal')
    return None

  def use_key(self, key):
    if key not in self.keys:
      self.keys.append(key)
    return key

  def check_attr(self, node, name):
    if self.kind == 'backdrop':
      self.refuse(node, 'attribute self.{} (a Backdrop has no registers; keep its state in '
                  'the_plot)'.format(name))
    reserved = _RESERVED.get(self.kind, ())
    if (name in reserved or hasattr(self.klass, name) or
        any(r.endswith('*') and name.startswith(r[:-1]) for r in reserved)):
      self.refuse(node, 'attribute self.{} (not an int or bool of this object)'.format(name))

  def use_attr(self, node, name, t='int'):
    """The register of attribute `name` holding a `t` ('int' or 'pos'; a position
    attribute's registers are ('attr', name, 0) and ('attr', name, 1))."""
    self.check_attr(node, name)
    have = self.attr_types.setdefault(name, t)
    if have != t:
      self.refuse(node, 'attribute self.{} holding a {} and a {}'.format(
          name, _TYPE_NAMES[have], _TYPE_NAMES[t]))
    if name not in self.attrs:
      self.attrs.append(name)
    return ('attr', name)

  def register_attr(self, node):
    """`name` of `self.name` when it is a register attribute, else None."""
    if (isinstance(node, ast.Attribute) and self.is_self(node.value) and
        node.attr not in _POSITIONS and node.attr not in ('corner', 'visible', 'Position') and
        not (self.kind == 'plain' and node.attr in _SPRITE_STATE)):
      return node.attr
    return None

  def claim_pos(self, node):
    """Where a position is needed: an attribute of no type yet becomes a position one."""
    name = self.register_attr(node)
    reserved = _RESERVED.get(self.kind, ())
    if (name is not None and name not in self.attr_types and name not in reserved and
        not hasattr(self.klass, name) and
        not any(r.endswith('*') and name.startswith(r[:-1]) for r in reserved)):
      self.use_attr(node, name, 'pos')

  def position_ctor(self, node):
    """(row, col) argument nodes of `Position(r, c)` / `Position(row=r, col=c)`, where
    Position is things.Sprite.Position as `self.Position` or through the module globals,
    else None."""
    if not isinstance(node, ast.Call):
      return None
    f = node.func
    if isinstance(f, ast.Attribute) and self.is_self(f.value) and f.attr == 'Position':
      fn = inspect.getattr_static(self.klass, 'Position', None)
    else:
      fn = self.callee(f)
    if fn is not things.Sprite.Position:
      return None
    args = dict(zip(('row', 'col'), node.args))
    for k in node.keywords:
      if k.arg not in ('row', 'col') or k.arg in args:
        self.refuse(node, 'these arguments of Position()')
      args[k.arg] = k.value
    if len(node.args) > 2 or set(args) != {'row', 'col'}:
      self.refuse(node, 'these arguments of Position()')
    return args['row'], args['col']

  def use_stream(self, stream):
    if stream not in self.streams:
      self.streams.append(stream)
    return ('rng', stream)

  def need(self, node, kinds, what):
    if self.kind not in kinds.split():
      self.refuse(node, '{} in a {} class'.format(what, self.kind))

  def number(self, node):
    """Value of an int / float literal, optionally negated, else None."""
    sign = 1
    if isinstance(node, ast.UnaryOp) and isinstance(node.op, ast.USub):
      sign, node = -1, node.operand
    if (isinstance(node, ast.Constant) and isinstance(node.value, (int, float)) and
        not isinstance(node.value, bool)):
      return sign * node.value
    return None

  # -------------------------------------------------------- inlined helpers
  def helper(self, node):
    """What a call of one of the game's own helpers runs, else None: for `self.name(...)`
    the attribute `name` of the entity's class along its MRO when it is the game's code
    (methods of this package's classes keep their own treatment), for `name(...)` a
    function of the game's code found through the module globals (`_user_code` decides
    both)."""
    if not isinstance(node, ast.Call):
      return None
    f = node.func
    if isinstance(f, ast.Attribute) and self.is_self(f.value):
      obj = inspect.getattr_static(self.klass, f.attr, None)
      self.methods[f.attr] = obj        # every resolution, for `registered` to compare
      fn = obj
      if isinstance(obj, property):
        fn = obj.fget
      elif isinstance(obj, (staticmethod, classmethod)):
        fn = obj.__func__
      return obj if isinstance(fn, types.FunctionType) and _user_code(fn) else None
    fn = self.callee(f)
    if isinstance(fn, types.FunctionType) and _user_code(fn):
      return fn
    return None

  def helper_type(self, node):
    """What the helper `node` calls returns ('int', 'pos', 'motion' or 'nothing'), found by
    inlining it into code that is thrown away; None when `node` calls no helper.  The
    call is then inlined again, so a chain of helpers each asked for its type costs up to
    2 ** depth inlines; MAX_HELPER_DEPTH bounds that at 256."""
    if self.helper(node) is None:
      return None
    if node not in self.helper_types:
      at = len(self.ir)
      self.helper_types[node] = self.inline(node)
      del self.ir[at:]
    return self.helper_types[node]

  def refuse_helper(self, fn, call, what):
    """Refuse the helper `fn` that `call`, in the function being compiled, runs."""
    site = (self.short, self.first + call.lineno - 1)
    self.callers.append(site)
    msg = '{}.{}, line {}: {} is not compiled{}'.format(
        fn.__module__, fn.__qualname__, fn.__code__.co_firstlineno, what, self.called_from())
    self.callers.pop()
    raise NotLoweredError(msg)

  def helper_def(self, obj, call):
    """(function, its def, source lines, first line) of the helper `obj`; refuses the forms
    that are not inlined."""
    fn = obj
    for kind in (staticmethod, classmethod, property):
      if isinstance(obj, kind):
        fn = obj.fget if kind is property else obj.__func__
        if isinstance(fn, types.FunctionType):
          self.refuse_helper(fn, call, 'a {} helper'.format(kind.__name__))
        self.refuse(call, 'the call {}()'.format(ast.unparse(call.func)))
    if fn.__name__ == '<lambda>':
      self.refuse_helper(fn, call, 'a lambda')
    if fn in self.active:
      cycle = self.active[self.active.index(fn):] + [fn]
      self.refuse_helper(fn, call, 'recursion ({})'.format(
          ' -> '.join(g.__qualname__ for g in cycle)))
    if len(self.active) >= MAX_HELPER_DEPTH:
      self.refuse_helper(fn, call, 'helpers nested more than {} deep'.format(MAX_HELPER_DEPTH))
    if fn.__code__.co_flags & (inspect.CO_GENERATOR | inspect.CO_COROUTINE |
                               inspect.CO_ASYNC_GENERATOR):
      self.refuse_helper(fn, call, 'a generator')
    free = [v for v in fn.__code__.co_freevars if v != '__class__']   # __class__: super()
    if free:
      self.refuse_helper(fn, call, 'a closure over {}'.format(', '.join(free)))
    try:
      lines, first = inspect.getsourcelines(fn)
    except (OSError, TypeError):
      self.refuse_helper(fn, call, 'a helper whose source is not available')
    fdef = ast.parse(textwrap.dedent(''.join(lines))).body[0]
    if not isinstance(fdef, ast.FunctionDef):
      self.refuse_helper(fn, call, type(fdef).__name__)
    if fdef.decorator_list:
      self.refuse_helper(fn, call, 'a decorated helper')
    a = fdef.args
    if a.vararg or a.kwarg or a.kwonlyargs:
      self.refuse_helper(fn, call, '*args, **kwargs or a keyword-only parameter')
    params = a.posonlyargs + a.args
    for p, d in zip(params[len(params) - len(a.defaults):], a.defaults):
      if not (type(self.number(d)) is int or isinstance(d, ast.Constant) and (
          d.value is None or type(d.value) is bool or (type(d.value) is str and len(d.value) == 1))):
        self.refuse_helper(fn, call, 'the default {}={}'.format(p.arg, ast.unparse(d)))
    return fn, fdef, lines, first

  def inline(self, call):
    """Emit the body of the helper `call` runs in place of the call.  Returns what it
    leaves on the stack: the type of its value, or 'nothing'."""
    fn, fdef, lines, first = self.helper_def(self.helper(call), call)
    what = '{}()'.format(ast.unparse(call.func))
    params = [p.arg for p in fdef.args.posonlyargs + fdef.args.args]
    defaults = dict(zip(params[len(params) - len(fdef.args.defaults):], fdef.args.defaults))
    role = {}
    if isinstance(call.func, ast.Attribute):       # a method: its first parameter is self
      if not params:
        self.refuse_helper(fn, call, 'a method without a self parameter')
      role[params.pop(0)] = 'self'
    bound = dict(zip(params, call.args))
    if len(call.args) > len(params) or any(isinstance(x, ast.Starred) for x in call.args):
      self.refuse(call, 'these arguments of ' + what)
    positional_only = {p.arg for p in fdef.args.posonlyargs}
    for k in call.keywords:
      if k.arg not in params or k.arg in bound or k.arg in positional_only:
        self.refuse(call, 'these arguments of ' + what)
      bound[k.arg] = k.value
    for p in params:
      if p not in bound and p not in defaults:
        self.refuse(call, '{} without its argument {}'.format(what, p))
    # Arguments in the caller's frame, left to right, then the defaults.
    n_slots, local, consts = self.n_slots, {}, {}
    for p in [p for p in bound] + [p for p in params if p not in bound]:
      arg = bound.get(p, defaults.get(p))
      if isinstance(arg, ast.Name) and self.role.get(arg.id) in _ROLES:
        role[p] = self.role[arg.id]
        continue
      if isinstance(arg, ast.Constant) and type(arg.value) is str and len(arg.value) == 1:
        consts[p] = arg.value
        continue
      if isinstance(arg, ast.Constant) and arg.value is None:
        self.emit('PUSH', 0)                        # None as a motion result
        t = 'motion'
      elif self.helper(arg) is not None or p not in bound:
        t = self.value(arg)
      else:
        try:
          t = self.value(arg)
        except NotLoweredError:                     # refused below, naming the argument
          t = None
      if t not in _WIDTH:
        self.refuse(call, 'the argument {}={} of {}'.format(p, ast.unparse(arg), what))
      slot = self.n_slots
      self.n_slots += _WIDTH[t]
      if self.n_slots > _lib.CODE_LOCALS:
        self.refuse(call, 'more than {} local slots'.format(_lib.CODE_LOCALS))
      for s in reversed(range(slot, self.n_slots)):
        self.emit('STORE', s)
      local[p] = (slot, t)
    # The helper's own frame.
    constants = _Constants(consts)
    body = [constants.visit(st) for st in fdef.body]
    saved = {k: getattr(self, k) for k in _FRAME}
    self.callers.append((self.short, self.first + call.lineno - 1))
    self.active.append(fn)
    self.lines, self.first, self.globals = lines, first, fn.__globals__
    self.role, self.locals, self.ret = role, local, _Return(self.label())
    self.where, self.short = '{}.{}'.format(fn.__module__, fn.__qualname__), fn.__qualname__
    try:
      if constants.stored is not None:
        self.refuse(constants.stored, 'assigning the argument ' + constants.stored.id)
      self.stmts(body)
      ret = self.ret
      if ret.type is not None and ret.bare:
        if ret.type != 'motion':
          self.refuse(ret.bare[0][1], 'a bare return in a helper that returns a ' +
                      _TYPE_NAMES[ret.type])
        for at, _ in reversed(ret.bare):         # None as a motion result
          self.ir.insert(at, ('PUSH', 0))
      if ret.type is not None and _falls_off(body):
        if ret.type != 'motion':
          self.refuse(fdef, 'a helper that returns a {} and can fall off its end'.format(
              _TYPE_NAMES[ret.type]))
        self.emit('PUSH', 0)
      # A jump to the label that immediately follows is not emitted.
      at = len(self.ir)
      while at and (self.ir[at - 1][0] == 'LABEL' or self.ir[at - 1] == ('JMP', ret.label)):
        if self.ir[at - 1][0] == 'JMP':
          del self.ir[at - 1]
        at -= 1
      self.place(ret.label)
      return ret.type or 'nothing'
    finally:
      for k, v in saved.items():
        setattr(self, k, v)
      self.callers.pop()
      self.active.pop()
      self.n_slots = n_slots

  def helper_return(self, st):
    """`return`, `return None`, `return <call returning None>` or `return <value>` in an
    inlined helper: a jump to its end, with the value on the stack."""
    ret, v = self.ret, st.value
    if v is None or (isinstance(v, ast.Constant) and v.value is None):
      t = None
    elif isinstance(v, ast.Call) and self.returns_nothing(v):
      self.call_stmt(v)
      t = None
    else:
      t = self.value(v)
      if t not in _WIDTH:
        self.refuse(st, 'returning a ' + _TYPE_NAMES[t])
    self.emit('JMP', ret.label)
    if t is None:
      ret.bare.append((len(self.ir) - 1, st))
    elif ret.type is None:
      ret.type = t
    elif ret.type != t:
      self.refuse(st, 'returning a {} and a {}'.format(_TYPE_NAMES[ret.type], _TYPE_NAMES[t]))

  def value(self, node):
    """Push a value a helper takes or returns: as expr(), and a tuple as a position."""
    if isinstance(node, ast.Tuple):
      self.pos(node, node)
      return 'pos'
    return self.expr(node)

  def returns_nothing(self, call):
    """Is `call` a statement call: a helper that returns nothing, `_teleport`, a Scrolly's
    motion helper or a `the_plot` method?"""
    f = call.func
    if self.helper(call) is not None:
      return self.helper_type(call) == 'nothing'
    if isinstance(f, ast.Attribute) and self.is_self(f.value):
      return f.attr == '_teleport' or (f.attr in _MOTIONS and self.kind == 'scrolly')
    return (isinstance(f, ast.Attribute) and self.is_param(f.value, 'the_plot') and
            f.attr in ('add_reward', 'terminate_episode', 'change_default_discount'))

  # ----------------------------------------------------------- statements
  def stmts(self, body):
    for st in body:
      self.stmt(st)

  def stmt(self, st):
    if isinstance(st, ast.Expr):
      v = st.value
      if isinstance(v, ast.Constant) and isinstance(v.value, str):
        return                                    # docstring
      if isinstance(v, ast.Call):
        return self.call_stmt(v)
      self.refuse(st, 'an expression statement')
    elif isinstance(st, ast.Pass):
      return
    elif isinstance(st, ast.Delete):
      if all(isinstance(t, ast.Name) for t in st.targets):
        return
      self.refuse(st, '`del` of anything but names')
    elif isinstance(st, ast.Return):
      if self.ret is not None:
        return self.helper_return(st)
      if st.value is not None and not (isinstance(st.value, ast.Constant) and
                                       st.value.value is None):
        self.refuse(st, 'returning a value')
      self.emit('RET')
    elif isinstance(st, ast.If):
      self.truth(st.test)
      other, end = self.label(), self.label()
      self.emit('JZ', other)
      self.stmts(st.body)
      if st.orelse:
        self.emit('JMP', end)
      self.place(other)
      if st.orelse:
        self.stmts(st.orelse)
        self.place(end)
    elif isinstance(st, ast.Assign):
      if len(st.targets) != 1:
        self.refuse(st, 'chained assignment')
      self.assign(st.targets[0], st.value, st)
    elif isinstance(st, ast.AugAssign):
      self.aug_assign(st)
    else:
      self.refuse(st, type(st).__name__)

  def local(self, name, t, st):
    """The first slot of local variable `name` holding a `t`."""
    if name in self.role:
      self.refuse(st, 'assigning an update() argument')
    if t == 'char':
      self.refuse(st, 'a character in a variable')
    slot, have = self.locals.get(name, (None, None))
    if have is None:
      slot = self.n_slots
      self.n_slots += 2 if t == 'pos' else 1
      if self.n_slots > _lib.CODE_LOCALS:
        self.refuse(st, 'more than {} local slots'.format(_lib.CODE_LOCALS))
      self.locals[name] = (slot, t)
    elif have != t:
      self.refuse(st, 'variable {} holding a {} and a {}'.format(
          name, _TYPE_NAMES[have], _TYPE_NAMES[t]))
    return slot

  def assign(self, target, value, st):
    if isinstance(target, ast.Name):
      if target.id in self.role:
        self.refuse(st, 'assigning an update() argument')
      t = self.expr(value)
      slot = self.local(target.id, t, st)
      if t == 'pos':
        self.emit('STORE', slot + 1)
      self.emit('STORE', slot)
      return
    if isinstance(target, ast.Tuple):
      # `r, c = <position>`
      names = target.elts
      if len(names) != 2 or not all(isinstance(n, ast.Name) for n in names):
        self.refuse(st, 'unpacking into anything but two names')
      if any(n.id in self.role for n in names):
        self.refuse(st, 'assigning an update() argument')
      if self.expr(value) != 'pos':
        self.refuse(st, 'unpacking something that is not a position')
      slots = [self.local(n.id, 'int', st) for n in names]
      self.emit('STORE', slots[1])
      self.emit('STORE', slots[0])
      return
    if isinstance(target, ast.Subscript) and self.is_self_curtain(target.value):
      if self.kind == 'backdrop':
        return self.backdrop_write(target.slice, value, st)
    if (isinstance(target, ast.Subscript) and isinstance(target.value, ast.Attribute) and
        target.value.attr == 'curtain' and self.is_param(target.value.value, 'backdrop')):
      self.refuse(st, "a write to backdrop.curtain (only the Backdrop's own update() writes it)")
    if isinstance(target, ast.Subscript) and self.pattern_owner(target.value) is not None:
      if self.pattern_owner(target.value) != -1:
        self.refuse(st, "a write to another entity's whole_pattern")
      if _sliced(target.slice):
        self.refuse(st, 'a whole_pattern slice')
      self.cell(target.slice, st)
      self.scalar(value)
      self.emit('SETPAT')
      return
    if isinstance(target, ast.Attribute) and self.is_self(target.value):
      if self.kind == 'plain' and target.attr == '_position':
        if isinstance(value, ast.Tuple):
          self.refuse(st, 'a bare tuple as a position (upstream its .row fails later; use '
                      'self.Position(row, col))')
        self.pos(value, st)
        self.emit('SETFIELD', _lib.FIELD_COL)
        self.emit('SETFIELD', _lib.FIELD_ROW)
        return
      if self.kind == 'plain' and target.attr == '_visible':
        self.truth(value)
        self.emit('SETFIELD', _lib.FIELD_VISIBLE)
        return
      self.check_attr(target, target.attr)
      if self.attr_types.get(target.attr) == 'pos':
        self.pos(value, st)
        t = 'pos'
      else:
        t = self.expr(value)
        if t not in ('int', 'pos'):
          self.refuse(value, 'a {} where a number is needed'.format(_TYPE_NAMES[t]))
      reg = self.use_attr(target, target.attr, t)
      if t == 'pos':
        self.emit('SETR', reg + (1,))
        self.emit('SETR', reg + (0,))
      else:
        self.emit('SETR', reg)
      return
    key = self.plot_key(target)
    if key is not None:
      self.scalar(value)
      self.emit('SETP', ('key', key))
      return
    if (isinstance(target, ast.Subscript) and isinstance(target.value, ast.Attribute) and
        self.is_self(target.value.value) and target.value.attr == 'curtain'):
      self.need(st, 'drape', 'a curtain write')   # a Scrolly's curtain is its pattern's
      sl = target.slice
      if isinstance(sl, ast.Slice):
        if sl.lower is not None or sl.upper is not None or sl.step is not None:
          self.refuse(st, 'a curtain slice other than [:]')
        self.scalar(value)
        self.emit('FILL')
      else:
        self.cell(sl, st)
        self.scalar(value)
        self.emit('SETCELL')
      return
    self.refuse(st, 'this assignment target')

  def aug_assign(self, st):
    op = _BINOPS.get(type(st.op))
    if op is None:
      self.refuse(st, 'augmented assignment ' + type(st.op).__name__)
    target = st.target
    if isinstance(target, ast.Attribute) and self.is_self(target.value):
      reg = self.use_attr(target, target.attr)
      load, store = ('GETR', reg), ('SETR', reg)
    elif self.plot_key(target) is not None:
      key = ('key', self.plot_key(target))
      load, store = ('GETP', key), ('SETP', key)
    elif isinstance(target, ast.Name) and self.locals.get(target.id, (0, None))[1] == 'int':
      slot = self.locals[target.id][0]
      load, store = ('LOAD', slot), ('STORE', slot)
    else:
      self.refuse(st, 'this augmented assignment target')
    self.emit(*load)
    self.scalar(st.value)
    self.emit(op)
    self.emit(*store)

  def call_stmt(self, call):
    f = call.func
    if self.helper(call) is not None:      # first: a game's override of a motion helper too
      t = self.inline(call)
      for _ in range(_WIDTH.get(t, 0)):       # a value used as a statement is discarded
        self.emit('POP')
      return
    if self.motion_choice(f):
      # `(self._east if c else self._west)(...)` as if / else
      other, end = self.label(), self.label()
      self.truth(f.test)
      self.emit('JZ', other)
      self.call_stmt(ast.copy_location(ast.Call(f.body, call.args, call.keywords), call))
      self.emit('JMP', end)
      self.place(other)
      self.call_stmt(ast.copy_location(ast.Call(f.orelse, call.args, call.keywords), call))
      self.place(end)
      return
    if (isinstance(f, ast.Attribute) and self.is_self(f.value) and f.attr in _MOTIONS and
        self.kind == 'scrolly'):
      if len(call.args) != 1 or call.keywords or not self.is_param(call.args[0], 'the_plot'):
        self.refuse(call, 'a Scrolly motion helper not called as (the_plot)')
      self.emit('SCROLL', _MOTIONS[f.attr])
      return
    if isinstance(f, ast.Attribute) and self.is_self(f.value) and f.attr in _MOTIONS:
      self.expr(call)
      self.emit('POP')
      return
    if isinstance(f, ast.Attribute) and self.is_self(f.value) and f.attr == '_teleport':
      self.need(call, 'sprite', '_teleport')
      if len(call.args) != 1 or call.keywords:
        self.refuse(call, '_teleport with other than one position')
      self.pos(call.args[0], call)
      self.emit('TELEPORT')
      return
    if isinstance(f, ast.Attribute) and self.is_param(f.value, 'the_plot'):
      if f.attr == 'add_reward' and len(call.args) == 1 and not call.keywords:
        arg = call.args[0]
        value = self.number(arg)
        if isinstance(value, float):
          self.float_reward = True
          self.emit('REWARD_F64', *_f64_halves(value))
        else:
          self.scalar(arg)
          self.emit('REWARD')
        return
      if f.attr in ('terminate_episode', 'change_default_discount'):
        args = list(call.args) + [k.value for k in call.keywords if k.arg == 'discount']
        if len(args) + len([k for k in call.keywords if k.arg != 'discount']) > 1:
          self.refuse(call, 'these arguments of ' + f.attr)
        if not args and f.attr == 'terminate_episode':
          value = 0.0
        else:
          value = self.number(args[0]) if args else None
        if value is None:
          self.refuse(call, 'a discount that is not a number literal')
        self.emit('TERMINATE' if f.attr == 'terminate_episode' else 'DISCOUNT', _f32_bits(value))
        return
    self.refuse(call, 'the call {}()'.format(ast.unparse(f)))

  # ----------------------------------------------------------- expressions
  def scalar(self, node):
    """An int (or bool) value."""
    t = self.expr(node)
    if t != 'int':
      self.refuse(node, 'a {} where a number is needed'.format(_TYPE_NAMES[t]))

  def truth(self, node):
    t = self.expr(node)
    if t not in ('int', 'motion'):
      self.refuse(node, 'a {} as a truth value'.format(_TYPE_NAMES[t]))

  def pos(self, node, where):
    self.claim_pos(node)
    parts = self.pos_parts(node)
    if parts is None:
      self.refuse(where, 'something that is not a position')
    for part in parts:
      part()

  def cell(self, node, where):
    """Push (row, col) of a cell index: [r, c] or a position."""
    if isinstance(node, ast.Tuple) and len(node.elts) == 2:
      self.scalar(node.elts[0])
      self.scalar(node.elts[1])
    else:
      self.pos(node, where)

  def pos_parts(self, node):
    """Two emitters (row, col) of a position expression, else None."""
    def field(ent, f):
      return lambda: self.emit('FIELD', ent, f)
    if self.is_shape(node):
      return (lambda: self.emit('PUSH', ('rows',)), lambda: self.emit('PUSH', ('cols',)))
    if isinstance(node, ast.Attribute):
      owner = None
      if self.is_self(node.value):
        owner = -1
      elif self.thing_char(node.value) is not None:
        owner = ('ent', self.thing_char(node.value))
      if owner is not None:
        if node.attr in _POSITIONS:
          if owner == -1:
            self.need(node, 'sprite plain' if node.attr == 'position' else 'sprite',
                      '.' + node.attr)
          return tuple(field(owner, f) for f in _POSITIONS[node.attr])
        if owner == -1 and self.kind == 'plain' and node.attr == '_position':
          return tuple(field(owner, f) for f in _POSITIONS['position'])
        name = self.register_attr(node)
        if name is not None and self.attr_types.get(name) == 'pos':
          reg = self.use_attr(node, name, 'pos')
          return (lambda: self.emit('GETR', reg + (0,)), lambda: self.emit('GETR', reg + (1,)))
        if node.attr == 'corner' and self.kind != 'backdrop':
          return (lambda: self.emit('PUSH', ('rows',)), lambda: self.emit('PUSH', ('cols',)))
    if isinstance(node, ast.Name) and self.locals.get(node.id, (0, None))[1] == 'pos':
      slot = self.locals[node.id][0]
      return (lambda: self.emit('LOAD', slot), lambda: self.emit('LOAD', slot + 1))
    if self.pattern_position(node) is not None:   # one call pushes both
      return (lambda: self.pattern_position(node, emit=True), lambda: None)
    if self.position_ctor(node) is not None:
      row, col = self.position_ctor(node)
      return (lambda: self.scalar(row), lambda: self.scalar(col))
    if isinstance(node, ast.Tuple) and len(node.elts) == 2:
      return (lambda: self.scalar(node.elts[0]), lambda: self.scalar(node.elts[1]))
    if self.helper_type(node) == 'pos':           # one inlined call pushes both
      return (lambda: self.inline(node), lambda: None)
    return None

  def component(self, node, index, where):
    parts = self.pos_parts(node)
    if parts is None or isinstance(node, ast.Tuple):
      self.refuse(where, 'indexing something that is not a position')
    if self.pattern_position(node) is not None or self.helper_type(node) == 'pos':
      parts[0]()
      if index == 1:                      # keep the column: through a fresh local slot
        slot = self.local(' tmp%d' % self.n_slots, 'int', where)
        self.emit('STORE', slot)
      self.emit('POP')
      if index == 1:
        self.emit('LOAD', slot)
      return 'int'
    parts[index]()
    return 'int'

  def expr(self, node):
    """Emit code pushing `node`'s value; returns its type: 'int' (bools too), 'pos'
    (two words), 'motion' (1 = blocked, 0 = None) or 'char' (chr of a cell)."""
    if isinstance(node, ast.Constant):
      if isinstance(node.value, (bool, int)):
        self.emit('PUSH', int(node.value))
        return 'int'
      self.refuse(node, 'the literal {!r} here'.format(node.value))
    if isinstance(node, ast.Name):
      if node.id in self.locals:
        slot, t = self.locals[node.id]
        self.emit('LOAD', slot)
        if t == 'pos':
          self.emit('LOAD', slot + 1)
        return t
      if self.role.get(node.id) == 'actions':
        self.refuse(node, '`actions` outside ==, != , in and `is None`')
      self.refuse(node, 'the name ' + node.id)
    if isinstance(node, ast.Attribute):
      return self.attribute(node)
    if isinstance(node, ast.Subscript):
      return self.subscript(node)
    if isinstance(node, ast.Call):
      return self.call(node)
    if isinstance(node, ast.BinOp):
      op = _BINOPS.get(type(node.op))
      if op is None:
        self.refuse(node, 'the operator ' + type(node.op).__name__)
      self.scalar(node.left)
      self.scalar(node.right)
      self.emit(op)
      return 'int'
    if isinstance(node, ast.UnaryOp):
      if isinstance(node.op, ast.USub):
        self.scalar(node.operand)
        self.emit('NEG')
      elif isinstance(node.op, ast.UAdd):
        self.scalar(node.operand)
      elif isinstance(node.op, ast.Not):
        self.truth(node.operand)
        self.emit('NOT')
      else:
        self.refuse(node, 'the operator ' + type(node.op).__name__)
      return 'int'
    if isinstance(node, ast.BoolOp):
      # Python's value semantics: `a or b` is a if a is true, else b.
      end, kinds = self.label(), set()
      for i, v in enumerate(node.values):
        t = self.expr(v)
        if t not in ('int', 'motion'):
          self.refuse(v, 'a {} in and / or'.format(_TYPE_NAMES[t]))
        kinds.add(t)
        if i < len(node.values) - 1:
          self.emit('DUP')
          self.emit('JZ' if isinstance(node.op, ast.And) else 'JNZ', end)
          self.emit('POP')
      self.place(end)
      return 'int' if kinds == {'int'} else 'motion'
    if isinstance(node, ast.IfExp):
      other, end = self.label(), self.label()
      self.truth(node.test)
      self.emit('JZ', other)
      t = self.expr(node.body)
      self.emit('JMP', end)
      self.place(other)
      if self.expr(node.orelse) != t or t == 'pos':
        self.refuse(node, 'a conditional expression over different or position values')
      self.place(end)
      return t
    if isinstance(node, ast.Compare):
      return self.compare(node)
    self.refuse(node, type(node).__name__)

  def attribute(self, node):
    ch = self.palette_char(node)
    if ch is not None:
      self.emit('PUSH', ('palette', ch))
      return 'int'
    if node.attr in ('row', 'col') and self.is_shape(node.value):
      self.refuse(node, 'the attribute .' + node.attr + ' of a shape')
    if self.pos_parts(node) is not None and not isinstance(node, ast.Tuple):
      for part in self.pos_parts(node):
        part()
      return 'pos'
    if node.attr in ('row', 'col'):
      return self.component(node.value, 0 if node.attr == 'row' else 1, node)
    if self.is_self(node.value):
      if node.attr == 'visible' or (self.kind == 'plain' and node.attr == '_visible'):
        self.need(node, 'sprite plain', '.visible')
        self.emit('FIELD', -1, _lib.FIELD_VISIBLE)
        return 'int'
      self.emit('GETR', self.use_attr(node, node.attr))
      return 'int'
    ch = self.thing_char(node.value)
    if ch is not None and node.attr == 'visible':
      self.emit('FIELD', ('ent', ch), _lib.FIELD_VISIBLE)
      return 'int'
    if self.is_param(node.value, 'the_plot') and node.attr == 'frame':
      self.emit('FRAME')
      return 'int'
    self.refuse(node, 'the attribute .' + node.attr)

  def owner(self, node):
    """-1 for `self`, ('ent', X) for `things['X']`, else None."""
    if self.is_self(node):
      return -1
    ch = self.thing_char(node)
    return None if ch is None else ('ent', ch)

  def pattern_owner(self, node):
    """-1 for `self.whole_pattern` (of a Scrolly), ('ent', X) for `things['X'].whole_pattern`,
    else None."""
    if isinstance(node, ast.Attribute) and node.attr == 'whole_pattern':
      owner = self.owner(node.value)
      if owner == -1:
        self.need(node, 'scrolly', 'self.whole_pattern')
      return owner
    return None

  def pattern_position(self, node, emit=False):
    """The opcode of `<scrolly>.pattern_position_prescroll / _postscroll(pos, the_plot)`,
    else None; `emit`: push the (row, col) it yields."""
    if not (isinstance(node, ast.Call) and isinstance(node.func, ast.Attribute) and
            node.func.attr in _PATTERN_POSITIONS):
      return None
    owner = self.owner(node.func.value)
    if owner is None or (owner == -1 and self.helper(node) is not None):
      return None
    if emit:
      if owner == -1:
        self.need(node, 'scrolly', node.func.attr)
      if (len(node.args) != 2 or node.keywords or
          not self.is_param(node.args[1], 'the_plot')):
        self.refuse(node, node.func.attr + ' not called as (position, the_plot)')
      self.pos(node.args[0], node)
      self.emit(_PATTERN_POSITIONS[node.func.attr], owner)
    return _PATTERN_POSITIONS[node.func.attr]

  def motion_choice(self, f):
    """Is callee `f` `(self._a if c else self._b)` over two motion helpers?"""
    return (isinstance(f, ast.IfExp) and
            all(isinstance(x, ast.Attribute) and self.is_self(x.value) and x.attr in _MOTIONS
                for x in (f.body, f.orelse)))

  def curtain_owner(self, node):
    """-1 for `self.curtain`, ('ent', X) for `things['X'].curtain`, else None."""
    if isinstance(node, ast.Attribute) and node.attr == 'curtain':
      if self.is_self(node.value):
        self.need(node, 'drape scrolly', 'self.curtain')
        return -1
      ch = self.thing_char(node.value)
      if ch is not None:
        return ('ent', ch)
    return None

  def subscript(self, node):
    key = self.plot_key(node)
    if key is not None:
      self.emit('GETP', ('key', key))
      return 'int'
    ch = self.palette_char(node)
    if ch is not None:
      self.emit('PUSH', ('palette', ch))
      return 'int'
    base, sl = node.value, node.slice
    if self.kind == 'backdrop' and self.is_self_curtain(base):   # its own live curtain
      if _sliced(sl):
        self.refuse(node, 'reading a curtain slice')
      self.cell(sl, node)
      self.emit('BACKDROP')
      return 'int'
    if self.is_param(base, 'board'):
      self.cell(sl, node)
      self.emit('BOARD')
      return 'int'
    if (isinstance(base, ast.Subscript) and self.is_param(base.value, 'layers') and
        isinstance(base.slice, ast.Constant) and isinstance(base.slice.value, str) and
        len(base.slice.value) == 1):
      self.cell(sl, node)
      self.emit('BOARD')
      self.emit('PUSH', ord(base.slice.value))
      self.emit('EQ')
      return 'int'
    if (isinstance(base, ast.Attribute) and base.attr == 'curtain' and
        self.is_param(base.value, 'backdrop')):
      self.cell(sl, node)
      self.emit('BACKDROP')
      return 'int'
    owner = self.pattern_owner(base)
    if owner is not None:
      if _sliced(sl):
        self.refuse(node, 'a whole_pattern slice')
      self.cell(sl, node)
      self.emit('PATTERN', owner)
      return 'int'
    owner = self.curtain_owner(base)
    if owner is not None:
      if isinstance(sl, ast.Slice):
        self.refuse(node, 'reading a curtain slice')
      self.cell(sl, node)
      self.emit('CURTAIN', owner)
      return 'int'
    if isinstance(sl, ast.Constant) and sl.value in (0, 1) and not isinstance(sl.value, bool):
      return self.component(base, sl.value, node)
    self.refuse(node, 'this subscript')

  def call(self, node):
    f = node.func
    if self.helper(node) is not None:      # first: a game's override of a motion helper too
      t = self.inline(node)
      if t == 'nothing':
        self.refuse(node, 'the value of {}(), which returns nothing'.format(ast.unparse(f)))
      return t
    if self.motion_choice(f):
      self.need(node, 'sprite', 'a motion result')
      return self.expr(ast.copy_location(ast.IfExp(
          f.test, ast.copy_location(ast.Call(f.body, node.args, node.keywords), node),
          ast.copy_location(ast.Call(f.orelse, node.args, node.keywords), node)), node))
    if self.pattern_position(node, emit=True) is not None:
      return 'pos'
    if self.position_ctor(node) is not None:
      for part in self.pos_parts(node):
        part()
      return 'pos'
    if isinstance(f, ast.Attribute) and self.is_self(f.value) and f.attr in _MOTIONS:
      self.need(node, 'sprite', f.attr)
      if (len(node.args) != 2 or node.keywords or not self.is_param(node.args[0], 'board') or
          not self.is_param(node.args[1], 'the_plot')):
        self.refuse(node, 'a motion helper not called as (board, the_plot)')
      self.emit('MOVE', _MOTIONS[f.attr])
      return 'motion'
    if isinstance(f, ast.Name) and len(node.args) == 1 and not node.keywords:
      arg = node.args[0]
      if f.id == 'int':
        self.scalar(arg)
        return 'int'
      if f.id == 'ord' and isinstance(arg, ast.Constant) and isinstance(arg.value, str) \
          and len(arg.value) == 1:
        self.emit('PUSH', ord(arg.value))
        return 'int'
      if f.id == 'chr':
        self.scalar(arg)
        return 'char'
    if (isinstance(f, ast.Attribute) and self.is_param(f.value, 'the_plot') and f.attr == 'get'
        and len(node.args) == 1 and not node.keywords and isinstance(node.args[0], ast.Constant)
        and isinstance(node.args[0].value, str)):
      self.emit('GETP', ('key', self.use_key(node.args[0].value)))
      return 'int'
    if isinstance(f, ast.Attribute) and f.attr == 'any' and not node.args and not node.keywords:
      owner = self.pattern_owner(f.value)
      if owner is not None:
        self.emit('PATANY', owner)
        return 'int'
      owner = self.curtain_owner(f.value)
      if owner is not None:
        self.emit('ANY', owner)
        return 'int'
    draw = self.generator_call(node)
    if draw is not None:
      self.draw(node, *draw)
      return 'int'
    self.refuse(node, 'the call {}()'.format(ast.unparse(f)))

  # ------------------------------------------------------------------ draws
  def callee(self, f):
    """What a name or a dotted chain through modules names in update()'s module (the
    `np.random.randint` of `np.random.randint(4)`), or None.  Only module attributes are
    looked up, so resolving runs no user code."""
    parts = []
    while isinstance(f, ast.Attribute):
      parts.append(f.attr)
      f = f.value
    if not isinstance(f, ast.Name) or f.id in self.role or f.id in self.locals:
      return None
    obj = self.globals.get(f.id)
    for name in reversed(parts):
      if isinstance(obj, types.ModuleType):
        obj = getattr(obj, name, None)
      elif isinstance(obj, type):            # a class attribute, looked up without running code
        obj = inspect.getattr_static(obj, name, None)
      else:
        return None
    return obj

  def generator_call(self, node):
    """(stream, kind) when `node` calls a function of a global generator, else None."""
    if not isinstance(node, ast.Call):
      return None
    fn = self.callee(node.func)
    for draw, stream, kind in _DRAWS:
      if fn is draw:
        return stream, kind
    return None

  def draw(self, node, stream, kind):
    """Emit the int draw `node` (generator_call's stream, kind); refuse other forms."""
    what = 'the call {}()'.format(ast.unparse(node.func))
    args, n = node.args, len(node.args)
    if (node.keywords or kind == 'float' or any(isinstance(a, ast.Starred) for a in args) or
        n not in {'randint': (1, 2) if stream == 'numpy' else (2,), 'randrange': (1, 2),
                  'choice': (1,)}[kind]):
      self.refuse(node, what)
    slot = self.use_stream(stream)
    rule = _lib.RAND_NUMPY if stream == 'numpy' else _lib.RAND_PYTHON
    if kind == 'choice' and isinstance(args[0], (ast.Tuple, ast.List)):
      values = [self.number(e) for e in args[0].elts]
      if not values or len(values) > 64 or not all(isinstance(v, int) for v in values):
        self.refuse(node, what)                 # empty, too long, or not int literals
      self.emit('PUSH', 0)
      self.emit('PUSH', len(values))
      self.emit('RANDINT', slot, rule)
      self.emit('PICK', len(values), *values)
      return
    if kind == 'choice':
      if stream == 'python':
        self.refuse(node, what)                 # random.choice takes a sequence
      self.emit('PUSH', 0)
      try:
        self.scalar(args[0])
      except NotLoweredError:
        self.refuse(node, what)                 # a sequence that is not a literal
    else:
      if n == 1:
        self.emit('PUSH', 0)
      for a in args:
        self.scalar(a)
      if kind == 'randint' and stream == 'python':
        rule = _lib.RAND_PYTHON_CLOSED
    self.emit('RANDINT', slot, rule)

  def float_draw(self, node, op, other, where):
    """`draw op other` for a float draw `node` and a number literal `other`."""
    what = 'the call {}()'.format(ast.unparse(node.func))
    value = self.number(other)
    if node.args or node.keywords or value is None or type(op) not in _CMPOPS:
      self.refuse(where, what)
    stream, _ = self.generator_call(node)
    self.emit('RANDCMP', self.use_stream(stream), list(_CMPOPS).index(type(op)),
              *_f64_halves(value))

  def literal_values(self, node, chars):
    """Codes of a literal tuple / list / string for `in`; `chars`: the left side is chr()."""
    if isinstance(node, ast.Constant) and isinstance(node.value, str):
      if not chars:
        self.refuse(node, '`in` a string on a number')
      return [ord(c) for c in node.value]
    if isinstance(node, (ast.Tuple, ast.List)):
      out = []
      for e in node.elts:
        if chars and isinstance(e, ast.Constant) and isinstance(e.value, str) and len(e.value) == 1:
          out.append(ord(e.value))
        elif not chars and self.number(e) is not None and isinstance(self.number(e), int):
          out.append(int(self.number(e)))
        elif not chars and isinstance(e, ast.Constant) and isinstance(e.value, bool):
          out.append(int(e.value))
        else:
          self.refuse(e, 'a non-literal or mismatched `in` element')
      if len(out) > 64:
        self.refuse(node, '`in` over more than 64 values')
      return out
    self.refuse(node, '`in` over something that is not a literal tuple, list or string')

  def compare(self, node):
    for x in [node.left] + node.comparators:
      if len(node.ops) > 1 and (self.generator_call(x) or (None, None))[1] == 'float':
        self.refuse(node, 'the call {}()'.format(ast.unparse(x.func)))   # drawn once, used twice
    if len(node.ops) == 1:
      self.compare1(node.left, node.ops[0], node.comparators[0], node)
      return 'int'
    end = self.label()
    left = node.left
    for i, (op, right) in enumerate(zip(node.ops, node.comparators)):
      self.compare1(left, op, right, node)
      if i < len(node.ops) - 1:
        self.emit('DUP')
        self.emit('JZ', end)
        self.emit('POP')
      left = right
    self.place(end)
    return 'int'

  def compare1(self, left, op, right, node):
    floats = [(self.generator_call(x) or (None, None))[1] == 'float' for x in (left, right)]
    if floats[0] and not floats[1]:
      return self.float_draw(left, op, right, node)
    if floats[1] and not floats[0]:
      return self.float_draw(right, _FLIPPED.get(type(op), ast.In)(), left, node)
    none = isinstance(right, ast.Constant) and right.value is None
    if isinstance(op, (ast.Is, ast.IsNot)):
      if not none:
        self.refuse(node, '`is` against anything but None')
      if self.is_param(left, 'actions'):
        self.emit('ACTION')
        self.emit('PUSH', _lib.ACTION_NONE)
      else:
        if self.expr(left) != 'motion':
          self.refuse(node, '`is None` on anything but `actions` and motion results')
        self.emit('PUSH', 0)
      self.emit('EQ' if isinstance(op, ast.Is) else 'NE')
      return
    if self.is_param(right, 'actions') and isinstance(op, (ast.Eq, ast.NotEq)):
      left, right = right, left
    if self.is_param(left, 'actions'):
      if isinstance(op, (ast.In, ast.NotIn)):
        values = self.literal_values(right, False)
        if any(v < 0 for v in values):
          self.refuse(node, 'a negative action')
        self.emit('ACTION')
        self.emit('IN', len(values), *values)
        if isinstance(op, ast.NotIn):
          self.emit('NOT')
        return
      if not isinstance(op, (ast.Eq, ast.NotEq)):
        self.refuse(node, 'an ordering comparison on `actions` (None on the first frame)')
      value = self.number(right)
      if value is None and isinstance(right, ast.Constant) and isinstance(right.value, bool):
        value = int(right.value)
      if not isinstance(value, int) or value < 0:
        self.refuse(node, '`actions` against anything but a non-negative int literal')
      self.emit('ACTION')
      self.emit('PUSH', value)
      self.emit('EQ' if isinstance(op, ast.Eq) else 'NE')
      return
    if isinstance(op, (ast.In, ast.NotIn)):
      t = self.expr(left)
      if t not in ('int', 'char'):
        self.refuse(node, '`in` on a ' + _TYPE_NAMES[t])
      values = self.literal_values(right, t == 'char')
      self.emit('IN', len(values), *values)
      if isinstance(op, ast.NotIn):
        self.emit('NOT')
      return
    name = _CMPOPS[type(op)]
    lp, rp = self.pos_parts(left), self.pos_parts(right)
    if lp is not None and rp is not None and name in ('EQ', 'NE') and not (
        isinstance(left, ast.Tuple) and isinstance(right, ast.Tuple)):
      for part in lp + rp:
        part()
      self.emit('EQ2')
      if name == 'NE':
        self.emit('NOT')
      return
    if (isinstance(right, ast.Constant) and isinstance(right.value, str) and
        len(right.value) == 1 and name in ('EQ', 'NE')):
      if self.expr(left) != 'char':
        self.refuse(node, 'a number compared with a string')
      self.emit('PUSH', ord(right.value))
      self.emit(name)
      return
    self.scalar(left)
    self.scalar(right)
    self.emit(name)


  # ------------------------------------------------------------- Backdrops
  def is_self_curtain(self, node):
    return isinstance(node, ast.Attribute) and node.attr == 'curtain' and self.is_self(node.value)

  def is_shape(self, node):
    """`board.shape`, or `self.curtain.shape` in a Backdrop: (rows, cols)."""
    return (isinstance(node, ast.Attribute) and node.attr == 'shape' and
            (self.is_param(node.value, 'board') or
             (self.kind == 'backdrop' and self.is_self_curtain(node.value))))

  def palette_char(self, node):
    """The character of `self.palette.X` / `self.palette['X']` in a Backdrop, its alias
    resolved (engine.py Palette), else None.  Lowering checks it against the palette."""
    if self.kind != 'backdrop':
      return None
    if isinstance(node, ast.Attribute):
      base, key = node.value, node.attr
    elif (isinstance(node, ast.Subscript) and isinstance(node.slice, ast.Constant) and
          isinstance(node.slice.value, str)):
      base, key = node.value, node.slice.value
    else:
      return None
    if not (isinstance(base, ast.Attribute) and base.attr == 'palette' and self.is_self(base.value)):
      return None
    return engine_lib.Palette._ALIASES.get(key, key)

  def is_byte(self, node):
    """Does `node` always lie in 0..255, so that NumPy stores it in a uint8 cell as it is?"""
    if isinstance(node, ast.Constant):
      return isinstance(node.value, bool) or (isinstance(node.value, int) and
                                               0 <= node.value <= 255)
    if self.palette_char(node) is not None:
      return True
    if (isinstance(node, ast.Call) and isinstance(node.func, ast.Name) and node.func.id == 'ord'
        and len(node.args) == 1 and isinstance(node.args[0], ast.Constant) and
        isinstance(node.args[0].value, str) and len(node.args[0].value) == 1):
      return ord(node.args[0].value) <= 255
    if isinstance(node, (ast.Compare, ast.UnaryOp)):
      return isinstance(node, ast.Compare) or isinstance(node.op, ast.Not)
    if isinstance(node, ast.Subscript) and not _sliced(node.slice):
      base = node.value
      return (self.is_param(base, 'board') or self.is_self_curtain(base) or
              (isinstance(base, ast.Attribute) and base.attr == 'curtain' and
               self.thing_char(base.value) is not None) or
              (isinstance(base, ast.Subscript) and self.is_param(base.value, 'layers')))
    return False

  def byte(self, node):
    """A value for a curtain cell: a form that lies in 0..255, or `x if c else y` of them.
    NumPy 2 raises OverflowError when a Python int outside 0..255 is stored in a uint8 cell
    but wraps a NumPy int; a device int32 does not say which it was, so no other int is
    written."""
    if isinstance(node, ast.IfExp):
      other, end = self.label(), self.label()
      self.truth(node.test)
      self.emit('JZ', other)
      self.byte(node.body)
      self.emit('JMP', end)
      self.place(other)
      self.byte(node.orelse)
      self.place(end)
      return
    if not self.is_byte(node):
      self.refuse(node, 'a curtain value that may lie outside 0..255 (write a palette '
                  "character, ord('c'), an int literal 0..255, a board or curtain cell or a bool)")
    self.scalar(node)

  def band(self, sl, where):
    """(lo, hi) of a band of rows `[a:b]` / `[a:b, :]` (None where omitted), or None for a
    cell index.  Refuses every other slice."""
    elts = sl.elts if isinstance(sl, ast.Tuple) else [sl]
    if not any(isinstance(x, ast.Slice) for x in elts):
      return None
    rows = elts[0]
    full = lambda x: (isinstance(x, ast.Slice) and x.lower is None and x.upper is None and
                      x.step is None)
    if not isinstance(rows, ast.Slice) or len(elts) > 2 or (len(elts) == 2 and not full(elts[1])):
      self.refuse(where, 'a row or column slice other than a band of rows [a:b, :]')
    if rows.step is not None:
      self.refuse(where, 'a stepped slice')
    out = []
    for bound in (rows.lower, rows.upper):
      value = None if bound is None else self.number(bound)
      if bound is not None and not isinstance(value, int):
        self.refuse(where, 'a slice bound that is not an int literal')
      out.append(value)
    return tuple(out)

  def roll(self, node, where):
    """(band, shift node, axis) of `np.roll(<curtain band>, shift, axis)`, else None."""
    if not (isinstance(node, ast.Call) and self.callee(node.func) is np.roll):
      return None
    args = dict(zip(('a', 'shift', 'axis'), node.args))
    for k in node.keywords:
      if k.arg not in ('shift', 'axis') or k.arg in args:
        self.refuse(where, 'these arguments of np.roll()')
      args[k.arg] = k.value
    if len(node.args) > 3 or 'shift' not in args:
      self.refuse(where, 'these arguments of np.roll()')
    axis = args.get('axis')
    if not (isinstance(axis, ast.Constant) and type(axis.value) is int and axis.value in (0, 1)):
      self.refuse(where, 'an np.roll axis that is not the literal 0 or 1')
    src = args['a']
    if self.is_self_curtain(src):
      band = (None, None)
    elif isinstance(src, ast.Subscript) and self.is_self_curtain(src.value):
      band = self.band(src.slice, where)
    else:
      band = None
    if band is None:
      self.refuse(where, "np.roll of something other than a band of the Backdrop's curtain")
    return band, args['shift'], axis.value

  def backdrop_write(self, sl, value, st):
    """`self.curtain[cell] = v`, `self.curtain[:] = v` or `self.curtain[band] =
    np.roll(self.curtain[band], shift, axis)` in a Backdrop's update()."""
    band = self.band(sl, st)
    if band is None:
      self.cell(sl, st)
      self.byte(value)
      self.emit('SETBACK')
      return
    rolled = self.roll(value, st)
    if rolled is not None:
      if rolled[0] != band:
        self.refuse(st, 'np.roll of another band than the one it is assigned to')
      self.scalar(rolled[1])
      self.emit('ROLLBACK', rolled[2], ('lo',) + band, ('hi',) + band)
      return
    if band != (None, None):
      self.refuse(st, 'a write to a band of rows other than np.roll of that band')
    self.byte(value)
    self.emit('FILLBACK')


class _Return(object):
  """The end of an inlined helper: its label, the type of the value it returns (None
  until a `return <value>`), and (IR index, node) of each `return` without a value."""

  def __init__(self, label):
    self.label, self.type, self.bare = label, None, []


class _Constants(ast.NodeTransformer):
  """A helper's body with each parameter bound to a one-character string literal read as
  that literal; `stored` is the first name node that assigns such a parameter."""

  def __init__(self, consts):
    self.consts, self.stored = consts, None

  def visit_Name(self, node):
    if node.id not in self.consts:
      return node
    if not isinstance(node.ctx, ast.Load):
      self.stored = self.stored or node
      return node
    return ast.copy_location(ast.Constant(self.consts[node.id]), node)


def _falls_off(body):
  """Can control reach the end of the statements `body`?"""
  if not body:
    return True
  last = body[-1]
  if isinstance(last, ast.Return):
    return False
  if isinstance(last, ast.If):
    return _falls_off(last.body) or _falls_off(last.orelse)
  return True


_STDLIB = tuple(os.path.realpath(sysconfig.get_paths()[k]) + os.sep
                for k in ('stdlib', 'platstdlib'))


def _user_code(fn):
  """Is the Python function `fn` the game's code, to be inlined?  One rule for methods
  and module functions: every function qualifies except this package's, NumPy's and the
  standard library's (by the file that defines it, so a game module named like a standard
  one, or a game installed as a package, qualifies).  A function of another library
  qualifies too, and compiles if its body lies in the subset."""
  if (fn.__module__ or '').split('.')[0] in ('numpy', 'pycolab_b200'):
    return False
  path = fn.__code__.co_filename
  if path.startswith('<frozen'):                 # standard modules frozen into Python
    return False
  path = os.path.realpath(path)
  return not (path.startswith(_STDLIB) and 'site-packages' not in path and
              'dist-packages' not in path)


def _sliced(index):
  """Does a subscript index take a slice on some axis?"""
  return any(isinstance(x, ast.Slice) for x in
             (index.elts if isinstance(index, ast.Tuple) else [index]))


# Attributes the prefabs keep for themselves (their state lives in the device records).
_RESERVED = {
    'sprite': {'_virtual_row', '_virtual_col', '_position', '_visible', '_prior_visible',
               '_c_h_a_r_a_c_t_e_r', '_c_o_r_n_e_r', '_impassable', '_confined_to_board',
               '_egocentric_scroller', '_scrolling_group'},
    'plain': {'_position', '_visible', '_c_h_a_r_a_c_t_e_r', '_c_o_r_n_e_r'},
    'drape': {'_c_u_r_t_a_i_n', '_c_h_a_r_a_c_t_e_r'},
    'scrolly': {'_c_u_r_t_a_i_n', '_c_h_a_r_a_c_t_e_r', '_w_h_o_l_e_p_a_t_t_e_r_n',
                '_northwest_corner', '_prescroll_northwest_corner', '_last_maybe_move_frame',
                '_northwest_corner_limit', '_scroll_margins', '_have_margins', '_board_shape',
                '_scrolling_group', '_pattern_at_init', '_margin_*'},
}


# ------------------------------------------------------------------ linking

def link(compiled, sprite_chars, drape_chars, rows, cols, plot_keys, rng_streams=(),
         backdrop=None):
  """Bytecode words for one game.  compiled: char -> `Compiled`; plot_keys: the key
  order of the plot registers; rng_streams: the generator of each RNG slot; backdrop: the
  `Compiled` of the Backdrop, whose entry goes in header word 1 + n (pcl.h program_arg[4]).
  Entities of one `Compiled` share their code: those of one class, and those of subclasses
  that inline the same helpers (`registered`)."""
  chars = list(sprite_chars) + list(drape_chars)
  S = len(sprite_chars)
  words = [len(chars)] + [0] * (len(chars) + (backdrop is not None))
  entry = {}
  for i, ch in enumerate(chars):
    comp = compiled[ch]
    if comp not in entry:
      entry[comp] = len(words)
      words += _encode(comp, len(words), chars, S, rows, cols, plot_keys, rng_streams)
    words[1 + i] = entry[comp]
  if backdrop is not None:
    words[1 + len(chars)] = len(words)
    words += _encode(backdrop, len(words), chars, S, rows, cols, plot_keys, rng_streams)
  if len(words) > _lib.MAX_CODE_WORDS:
    raise NotLoweredError('the compiled game needs {} code words, more than {}'.format(
        len(words), _lib.MAX_CODE_WORDS))
  return np.array(words, dtype=np.int32)


def _encode(comp, base, chars, S, rows, cols, plot_keys, rng_streams):
  addr, pc = {}, base
  for ins in comp.ir:                 # pass 1: label addresses
    if ins[0] == 'LABEL':
      addr[ins[1]] = pc
    else:
      pc += len(ins)

  def resolve(x, op):
    if not isinstance(x, tuple):
      return int(x)
    if x[0] == 'label':
      return addr[x[1]]
    if x[0] == 'attr':                # ('attr', name) or ('attr', name, half) of a position
      return comp.slot(x[1]) + (x[2] if len(x) > 2 else 0)
    if x[0] == 'key':
      return plot_keys.index(x[1])
    if x[0] == 'rng':
      return list(rng_streams).index(x[1])
    if x[0] == 'rows':
      return rows
    if x[0] == 'cols':
      return cols
    if x[0] == 'palette':             # lowering checked it against the game's palette
      return ord(x[1])
    if x[0] in ('lo', 'hi'):          # a band of rows, clipped as a Python slice
      lo, hi, _ = slice(x[1], x[2]).indices(rows)
      return lo if x[0] == 'lo' else max(lo, hi)
    ch = x[1]                         # ('ent', ch)
    if ch not in chars:
      raise NotLoweredError('{}: things[{!r}] names no entity of the game'.format(
          _name(comp.klass), ch))
    k = chars.index(ch)
    if (op == 'FIELD') != (k < S):     # FIELD names a sprite; the others a drape / Scrolly
      raise NotLoweredError('{}: things[{!r}] is not a {}'.format(
          _name(comp.klass), ch, 'sprite' if op == 'FIELD' else 'drape'))
    return k

  out = []
  for ins in comp.ir:                 # pass 2: words
    if ins[0] != 'LABEL':
      out.append(_lib.OP[ins[0]])
      out += [resolve(x, ins[0]) for x in ins[1:]]
  return out
