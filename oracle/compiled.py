"""CPU interpreter of the compiled program's bytecode (include/pcl.h PCL_OP_*).  TEST
INFRASTRUCTURE ONLY; nothing under `pycolab_b200/` imports it.

`make_world(game)` builds an `engine_model.World` from a lowered game of the compiled
program (`pycolab_b200.programs.compiled.lower`: its templates, registers and code words).
`compiled_program(world, ch, actions)` runs entity `ch`'s update(), and
`backdrop_program(world, actions)` the Backdrop's, by interpreting the same words the
device runs, one instruction at a time, over the oracle's registers: one loop for every
opcode, as csrc/compiled.cu's run_update is one.  The Python reference semantics it
restates: NumPy cell indexing, floor `//` and `%`, rewards summed in call order as Python
sums them (an int sum stays int), the Plot directives of plot.py:176-260, MazeWalker motion
(sprites.py:315-546) and the Scrolly prefab (drapes.py:293-659), the last two via
engine_model rather than restated here.

  - A Scrolly's curtain is engine_model's: the window of its pattern as of its last motion
    helper.  A postscroll query before the Scrolly moved raises RuntimeError, as upstream
    does; the device latches PCL_ENV_ERR_POSTSCROLL.
  - A plain Sprite (program_arg[3]) is an engine_model walker whose row, col and visible
    SETFIELD sets.  engine_model's render paints it with NumPy indexing: a negative index
    counts from the end once, and a visible sprite still off the board raises IndexError,
    as upstream's render does (rendering.py:139).  The device latches PCL_ENV_ERR_INDEX.
  - A compiled Backdrop (program_arg[4]) runs before update group 0 on the board of the
    last render (engine.py:718-723), and every render paints `world.backdrop`, which
    SETBACK / FILLBACK / ROLLBACK write as a cell write, a fill and np.roll of a band of
    rows.

Draws from the global generators (PCL_OP_RANDINT, RANDCMP, PICK) are restated from the
625 MT19937 words (624 key words + position), with the algorithms the device runs, rather
than by calling NumPy or `random`: test_drawn.py pins the restatement against the real
generators, and the oracle then shows that the words the device continues give what the
generators would.
"""

import struct

import numpy as np

from oracle import engine_model as em
from pycolab_b200 import _lib, lowering

OP = _lib.OP
_BINARY = {'ADD': lambda x, y: x + y, 'SUB': lambda x, y: x - y, 'MUL': lambda x, y: x * y,
           'FLOORDIV': lambda x, y: x // y, 'MOD': lambda x, y: x % y,
           'EQ': lambda x, y: x == y, 'NE': lambda x, y: x != y, 'LT': lambda x, y: x < y,
           'LE': lambda x, y: x <= y, 'GT': lambda x, y: x > y, 'GE': lambda x, y: x >= y}
_CMP = ('EQ', 'NE', 'LT', 'LE', 'GT', 'GE')


def _wrap32(x):
  return (int(x) + 2 ** 31) % 2 ** 32 - 2 ** 31


def _f32(bits):
  return float(struct.unpack('<f', struct.pack('<i', bits))[0])


def _f64(lo, hi):
  return struct.unpack('<d', struct.pack('<ii', lo, hi))[0]


# ------------------------------------------------------------------ MT19937
def _twist(mt):
  for j in range(624):
    y = (mt[j] & 0x80000000) | (mt[(j + 1) % 624] & 0x7fffffff)
    mt[j] = mt[(j + 397) % 624] ^ (y >> 1) ^ (0x9908b0df if y & 1 else 0)


def next32(mt):
  """One tempered output; mt[624] is the position."""
  if mt[624] >= 624:
    _twist(mt)
    mt[624] = 0
  y = mt[mt[624]]
  mt[624] += 1
  y ^= y >> 11
  y ^= (y << 7) & 0x9d2c5680
  y ^= (y << 15) & 0xefc60000
  return y ^ (y >> 18)


def numpy_below(mt, n):
  """RandomState.randint(0, n), 1 <= n < 2^32: masked rejection, no output for n == 1."""
  if n == 1:
    return 0
  mask = (1 << (n - 1).bit_length()) - 1
  while True:
    v = next32(mt) & mask
    if v < n:
      return v


def python_below(mt, n):
  """Random._randbelow(n), 1 <= n <= 2^32: getrandbits(n.bit_length()) until < n."""
  k = n.bit_length()
  while True:
    if k <= 32:
      r = next32(mt) >> (32 - k)
    else:
      lo = next32(mt)
      r = lo | (next32(mt) >> 31) << 32
    if r < n:
      return r


def random53(mt):
  """NumPy's random_sample() and Python's random(): 53 bits of two outputs."""
  a, b = next32(mt) >> 5, next32(mt) >> 6
  return (a * 67108864.0 + b) * (1.0 / 9007199254740992.0)


def randint(mt, rule, low, high):
  """PCL_OP_RANDINT: the drawn int, or None for an empty range (nothing consumed)."""
  width = high - low + (1 if rule == _lib.RAND_PYTHON_CLOSED else 0)
  if width <= 0:
    return None
  return low + (numpy_below(mt, width) if rule == _lib.RAND_NUMPY else python_below(mt, width))


def seeded_words(game, seed):
  """One list of words per RNG slot of `game`, seeded as BatchedEngine seeds env `seed`."""
  from pycolab_b200 import batched
  return [[int(w) for w in batched._mt_state(s, seed)] for s in game.rng_streams]


# ------------------------------------------------------------------ worlds
def make_world(game, words=None):
  """A fresh oracle env (the its_showtime() state) of lowered compiled game `game`.

  Each entity's `regs` are the record words its GETR / SETR k address, as run_update
  places them: a walker's AUX0-AUX2 (an egocentric one's from AUX2, its permits filling
  AUX0 / AUX1, which engine_model keeps apart), a plain Sprite's VROW, VCOL and AUX0-AUX2
  (the device skips FLAGS), a Scrolly's AUX0 onwards, a plain drape's whole record.

  `words`: for a game that draws, one mutable list of 625 ints per RNG slot
  (`game.rng_streams` order).  It is kept, not copied, so a trajectory that makes a new
  world per episode continues the same words, as the device does across auto-resets."""
  rows, cols = game.rows, game.cols
  ents = {}
  for s, ch in enumerate(game.sprite_chars):
    rec = [int(x) for x in game.sprites[s]]
    ego = bool(game.egocentric[s])
    w = em.Walker(ch, (rows, cols), (rec[_lib.S_ROW], rec[_lib.S_COL]),
                  confined=bool(game.confined[s]), egocentric=ego)
    w.vrow, w.vcol = rec[_lib.S_VROW], rec[_lib.S_VCOL]
    w.visible = bool(rec[_lib.S_FLAGS] & 1)
    w.prior_visible = (None, False, True)[(rec[_lib.S_FLAGS] >> 1) & 3]
    mask = game.impassable[s]
    w.impassable = frozenset(c for c in range(128) if (mask[c >> 5] >> (c & 31)) & 1)
    if (game.program_arg[3] >> s) & 1:
      w.regs = rec[_lib.S_VROW:_lib.S_FLAGS] + rec[_lib.S_AUX0:]
    else:
      w.regs = rec[_lib.S_AUX2 if ego else _lib.S_AUX0:]
    ents[ch] = w
  for d, ch in enumerate(game.drape_chars):
    rec = [int(x) for x in game.drapes[d]]
    if game.drape_kind[d]:
      margins = None if tuple(game.margins[d]) == (-1, -1) else tuple(game.margins[d])
      pattern = lowering.unpack_rows(game.patterns[d], game.pattern_cols)[:game.pattern_rows]
      drape = em.Scrolly(ch, (rows, cols), pattern,
                         (rec[_lib.D_CORNER_R], rec[_lib.D_CORNER_C]), margins=margins)
      drape.regs = rec[_lib.D_AUX0:]
    else:
      drape = em.PlainDrape(ch, lowering.unpack_rows(game.bits[d], cols)[:rows])
      drape.regs = rec
    ents[ch] = drape
  world = em.World(rows, cols, game.backdrop[:, :cols], ents, game.z_order,
                   [list(g) for g in game.groups], compiled_program)
  if game.program_arg[4]:
    world.backdrop_program = backdrop_program
  world.code = [int(x) for x in game.code]
  world.entity_chars = game.sprite_chars + game.drape_chars
  world.plot.regs = [int(x) for x in game.plot[_lib.P_AUX0:_lib.P_AUX0 + 4]]
  world.error = 0
  world.rng = words
  return world


# ------------------------------------------------------------------ the interpreter
def compiled_program(world, ch, actions):
  """Entity `ch`'s update(): its function, from header word 1 + its index."""
  _run(world, world.code[1 + world.entity_chars.index(ch)], world.things[ch], actions)


def backdrop_program(world, actions):
  """The Backdrop's update(): the function from header word 1 + n.  It has no registers
  and no entity of its own, so only the opcodes pcl_bind_code accepts there reach it."""
  _run(world, world.code[1 + len(world.entity_chars)], None, actions)


def _run(world, pc, me, actions):
  """Run the words from `pc` to their RET; `me` is the updated entity (None: the Backdrop)."""
  code, plot, chars = world.code, world.plot, world.entity_chars
  action = _lib.ACTION_NONE if actions is None else int(actions)
  stack, local = [], [0] * _lib.CODE_LOCALS
  board = (world.rows, world.cols)

  def ent(k):
    return me if k < 0 else world.things[chars[k]]

  def cell(r, c, shape):
    """NumPy's index rule over `shape`, or None (the device latches PCL_ENV_ERR_INDEX)."""
    r = r + shape[0] if r < 0 else r
    c = c + shape[1] if c < 0 else c
    if 0 <= r < shape[0] and 0 <= c < shape[1]:
      return r, c
    world.error |= _lib.ENV_ERR_INDEX
    return None

  while True:
    op = code[pc]
    name = _lib.OPS[op]
    a = code[pc + 1] if pc + 1 < len(code) else 0
    nxt = pc + 1 + _lib.OPERANDS[op]
    if name == 'RET':
      return
    # ---- stack, locals and control
    elif name == 'PUSH':
      stack.append(a)
    elif name == 'POP':
      stack.pop()
    elif name == 'DUP':
      stack.append(stack[-1])
    elif name == 'LOAD':
      stack.append(local[a])
    elif name == 'STORE':
      local[a] = stack.pop()
    elif name == 'JMP':
      nxt = a
    elif name in ('JZ', 'JNZ'):
      if (stack.pop() == 0) == (name == 'JZ'):
        nxt = a
    # ---- arithmetic
    elif name in _BINARY:
      y, x = stack.pop(), stack.pop()
      if name in ('FLOORDIV', 'MOD') and y == 0:
        world.error |= _lib.ENV_ERR_ARITH
        v = 0
      else:
        v = _BINARY[name](x, y)
      stack.append(_wrap32(v))
    elif name == 'NEG':
      stack.append(_wrap32(-stack.pop()))
    elif name == 'NOT':
      stack.append(int(stack.pop() == 0))
    elif name == 'EQ2':
      c2, r2, c1, r1 = stack.pop(), stack.pop(), stack.pop(), stack.pop()
      stack.append(int(r1 == r2 and c1 == c2))
    elif name in ('IN', 'PICK'):
      values = code[pc + 2:pc + 2 + a]
      x = stack.pop()
      if name == 'IN':
        stack.append(int(x in values))
      elif 0 <= x < a:
        stack.append(values[x])
      else:
        world.error |= _lib.ENV_ERR_INDEX
        stack.append(0)
      nxt += a
    # ---- draws from the global generators
    elif name == 'RANDINT':
      high, low = stack.pop(), stack.pop()
      v = randint(world.rng[a], code[pc + 2], low, high)
      if v is None:
        world.error |= _lib.ENV_ERR_RANGE
        v = low
      stack.append(v)
    elif name == 'RANDCMP':
      x, y = random53(world.rng[a]), _f64(code[pc + 3], code[pc + 4])
      stack.append(int(_BINARY[_CMP[code[pc + 2]]](x, y)))
    # ---- entities, registers and the Plot
    elif name == 'ACTION':
      stack.append(action)
    elif name == 'FRAME':
      stack.append(plot.frame)
    elif name == 'FIELD':
      w = ent(a)
      stack.append((w.row, w.col, w.vrow, w.vcol, int(bool(w.visible)))[code[pc + 2]])
    elif name == 'SETFIELD':
      v = stack.pop()
      if a == _lib.FIELD_VISIBLE:
        me.visible = v != 0
      else:
        setattr(me, 'row' if a == _lib.FIELD_ROW else 'col', v)
    elif name == 'GETR':
      stack.append(me.regs[a])
    elif name == 'SETR':
      me.regs[a] = stack.pop()
    elif name == 'GETP':
      stack.append(plot.regs[a])
    elif name == 'SETP':
      plot.regs[a] = stack.pop()
    # ---- board, backdrop and curtains
    elif name in ('BOARD', 'BACKDROP', 'CURTAIN'):
      c, r = stack.pop(), stack.pop()
      at = cell(r, c, board)
      if at is None:
        stack.append(0)
      elif name == 'BOARD':
        stack.append(int(world.board[at]))
      elif name == 'BACKDROP':
        stack.append(int(world.backdrop[at]))
      else:
        stack.append(int(ent(a).curtain[at]))
    elif name == 'SETCELL':
      v, c, r = stack.pop(), stack.pop(), stack.pop()
      at = cell(r, c, board)
      if at is not None:
        me.curtain[at] = v != 0
    elif name == 'FILL':
      me.curtain[:] = stack.pop() != 0
    elif name == 'ANY':
      stack.append(int(ent(a).curtain.any()))
    # ---- walker motion, through engine_model
    elif name == 'MOVE':
      stack.append(0 if em.walker_move(me, world.board, plot, a) is None else 1)
    elif name == 'TELEPORT':
      c, r = stack.pop(), stack.pop()
      em.walker_teleport(me, r, c)
    # ---- Scrollys, through engine_model
    elif name == 'SCROLL':
      em.scrolly_move(me, world, a)
    elif name in ('PRESCROLL', 'POSTSCROLL'):
      c, r = stack.pop(), stack.pop()
      fn = em.scrolly_prescroll if name == 'PRESCROLL' else em.scrolly_postscroll
      stack.extend(_wrap32(x) for x in fn(ent(a), (r, c), plot))
    elif name == 'PATTERN':
      c, r = stack.pop(), stack.pop()
      pattern = ent(a).pattern
      at = cell(r, c, pattern.shape)
      stack.append(0 if at is None else int(pattern[at]))
    elif name == 'SETPAT':
      v, c, r = stack.pop(), stack.pop(), stack.pop()
      at = cell(r, c, me.pattern.shape)
      if at is not None:
        me.pattern[at] = v != 0
    elif name == 'PATANY':
      stack.append(int(ent(a).pattern.any()))
    # ---- the Backdrop's curtain
    elif name == 'SETBACK':
      v, c, r = stack.pop(), stack.pop(), stack.pop()
      at = cell(r, c, board)
      if at is not None:
        world.backdrop[at] = v & 0xff
    elif name == 'FILLBACK':
      world.backdrop[:] = stack.pop() & 0xff
    elif name == 'ROLLBACK':
      lo, hi = code[pc + 2], code[pc + 3]
      world.backdrop[lo:hi] = np.roll(world.backdrop[lo:hi], stack.pop(), axis=a)
    # ---- Plot directives
    elif name == 'REWARD':
      plot.add_reward(stack.pop())
    elif name == 'REWARD_F64':
      plot.add_reward(_f64(a, code[pc + 2]))
    elif name == 'TERMINATE':
      plot.terminate_episode(_f32(a))
    elif name == 'DISCOUNT':
      plot.discount = _f32(a)
    else:
      raise AssertionError('opcode %d' % op)
    pc = nxt


def instructions(code, start, end):
  """Word indices of the instructions in [start, end); IN and PICK skip their value words."""
  out, pc = [], start
  while pc < end:
    out.append(pc)
    op = code[pc]
    pc += 1 + _lib.OPERANDS[op] + (code[pc + 1] if op in (OP['IN'], OP['PICK']) else 0)
  return out
