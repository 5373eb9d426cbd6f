"""CPU interpreter of compiled scrolling games: the compiled program's bytecode
(include/pcl.h PCL_OP_*) over `oracle.engine_model` worlds with Scrollys and egocentric
MazeWalkers.  TEST INFRASTRUCTURE ONLY.

`oracle/compiled.py` interprets the bytecode of walkers and plain drapes; this module runs
the same instruction set plus the Scrolly opcodes (SCROLL, PRESCROLL, POSTSCROLL, PATTERN,
SETPAT, PATANY), whose semantics it takes from engine_model's restatement of the prefab
(`scrolly_move`, `scrolly_prescroll`, `scrolly_postscroll`, egocentric `walker_move`)
rather than restating them.  A Scrolly's curtain is engine_model's: the window of its
pattern as of its last motion helper.  A postscroll query before the Scrolly moved raises
RuntimeError here, as upstream does; the device latches PCL_ENV_ERR_POSTSCROLL.

`make_world(game)` builds a fresh env of a lowered game of the compiled program; every
other opcode is interpreted as `oracle.compiled.compiled_program` does, with its draw and
bit helpers.
"""

from oracle import compiled as oc
from oracle import engine_model as em
from pycolab_b200 import _lib, lowering

_ERR_INDEX, _ERR_ARITH, _ERR_RANGE = 0x8, 0x20, 0x40
_BINARY = {'ADD': lambda x, y: x + y, 'SUB': lambda x, y: x - y, 'MUL': lambda x, y: x * y,
           'FLOORDIV': lambda x, y: x // y, 'MOD': lambda x, y: x % y,
           'EQ': lambda x, y: x == y, 'NE': lambda x, y: x != y, 'LT': lambda x, y: x < y,
           'LE': lambda x, y: x <= y, 'GT': lambda x, y: x > y, 'GE': lambda x, y: x >= y}
_CMP = ('EQ', 'NE', 'LT', 'LE', 'GT', 'GE')


def make_world(game, words=None):
  """A fresh oracle env (the its_showtime() state) of lowered compiled game `game`, its
  Scrollys and egocentric walkers included.  `words`: as oracle.compiled.make_world."""
  rows, cols = game.rows, game.cols
  ents = {}
  for s, ch in enumerate(game.sprite_chars):
    rec = game.sprites[s]
    ego = bool(game.egocentric[s])
    w = em.Walker(ch, (rows, cols), (int(rec[_lib.S_ROW]), int(rec[_lib.S_COL])),
                  confined=bool(game.confined[s]), egocentric=ego)
    w.vrow, w.vcol = int(rec[_lib.S_VROW]), int(rec[_lib.S_VCOL])
    w.visible = bool(rec[_lib.S_FLAGS] & 1)
    w.prior_visible = (None, False, True)[(int(rec[_lib.S_FLAGS]) >> 1) & 3]
    mask = game.impassable[s]
    w.impassable = frozenset(c for c in range(128) if (mask[c >> 5] >> (c & 31)) & 1)
    # an egocentric walker's AUX0 / AUX1 are its permits (engine_model keeps them apart)
    w.regs = [int(x) for x in rec[_lib.S_AUX2 if ego else _lib.S_AUX0:]]
    ents[ch] = w
  for d, ch in enumerate(game.drape_chars):
    rec = game.drapes[d]
    if game.drape_kind[d]:
      margins = None if tuple(game.margins[d]) == (-1, -1) else tuple(game.margins[d])
      pattern = lowering.unpack_rows(game.patterns[d], game.pattern_cols)[:game.pattern_rows]
      drape = em.Scrolly(ch, (rows, cols), pattern,
                         (int(rec[_lib.D_CORNER_R]), int(rec[_lib.D_CORNER_C])), margins=margins)
      drape.regs = [int(x) for x in rec[_lib.D_AUX0:]]
    else:
      drape = em.PlainDrape(ch, lowering.unpack_rows(game.bits[d], cols)[:rows])
      drape.regs = [int(x) for x in rec]
    ents[ch] = drape
  world = em.World(rows, cols, game.backdrop[:, :cols], ents, game.z_order,
                   [list(g) for g in game.groups], program)
  world.code = [int(x) for x in game.code]
  world.entity_chars = game.sprite_chars + game.drape_chars
  world.plot.regs = [int(x) for x in game.plot[_lib.P_AUX0:_lib.P_AUX0 + 4]]
  world.error = 0
  world.rng = words
  return world


def program(world, ch, actions):
  """Entity `ch`'s update(): its compiled words, one instruction at a time."""
  code, plot = world.code, world.plot
  chars = world.entity_chars
  me = world.things[ch]
  action = _lib.ACTION_NONE if actions is None else int(actions)
  stack, local = [], [0] * _lib.CODE_LOCALS
  pc = code[1 + chars.index(ch)]

  def ent(k):
    return me if k < 0 else world.things[chars[k]]

  def cell(r, c, shape):
    """NumPy's index rule over `shape`, or None (the device latches PCL_ENV_ERR_INDEX)."""
    r = r + shape[0] if r < 0 else r
    c = c + shape[1] if c < 0 else c
    if 0 <= r < shape[0] and 0 <= c < shape[1]:
      return r, c
    world.error |= _ERR_INDEX
    return None

  while True:
    op = code[pc]
    name = _lib.OPS[op]
    a = code[pc + 1] if pc + 1 < len(code) else 0
    nxt = pc + 1 + _lib.OPERANDS[op]
    if name == 'RET':
      return
    # ---- the Scrolly opcodes, through engine_model
    elif name == 'SCROLL':
      em.scrolly_move(me, world, a)
    elif name in ('PRESCROLL', 'POSTSCROLL'):
      c, r = stack.pop(), stack.pop()
      fn = em.scrolly_prescroll if name == 'PRESCROLL' else em.scrolly_postscroll
      stack.extend(oc._wrap32(x) for x in fn(ent(a), (r, c), plot))
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
    # ---- the others, as oracle/compiled.py interprets them
    elif name == 'RANDINT':
      high, low = stack.pop(), stack.pop()
      v = oc.randint(world.rng[a], code[pc + 2], low, high)
      if v is None:
        world.error |= _ERR_RANGE
        v = low
      stack.append(v)
    elif name == 'RANDCMP':
      x, y = oc.random53(world.rng[a]), oc._f64(code[pc + 3], code[pc + 4])
      stack.append(int(_BINARY[_CMP[code[pc + 2]]](x, y)))
    elif name in ('PICK', 'IN'):
      values = code[pc + 2:pc + 2 + a]
      x = stack.pop()
      if name == 'IN':
        stack.append(int(x in values))
      elif 0 <= x < a:
        stack.append(values[x])
      else:
        world.error |= _ERR_INDEX
        stack.append(0)
      nxt += a
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
    elif name in _BINARY:
      y, x = stack.pop(), stack.pop()
      if name in ('FLOORDIV', 'MOD') and y == 0:
        world.error |= _ERR_ARITH
        v = 0
      else:
        v = _BINARY[name](x, y)
      stack.append(oc._wrap32(v))
    elif name == 'NEG':
      stack.append(oc._wrap32(-stack.pop()))
    elif name == 'NOT':
      stack.append(int(stack.pop() == 0))
    elif name == 'EQ2':
      c2, r2, c1, r1 = stack.pop(), stack.pop(), stack.pop(), stack.pop()
      stack.append(int(r1 == r2 and c1 == c2))
    elif name == 'ACTION':
      stack.append(action)
    elif name == 'FRAME':
      stack.append(plot.frame)
    elif name == 'FIELD':
      w = ent(a)
      stack.append((w.row, w.col, w.vrow, w.vcol, int(bool(w.visible)))[code[pc + 2]])
    elif name == 'GETR':
      stack.append(me.regs[a])
    elif name == 'SETR':
      me.regs[a] = stack.pop()
    elif name == 'GETP':
      stack.append(plot.regs[a])
    elif name == 'SETP':
      plot.regs[a] = stack.pop()
    elif name in ('BOARD', 'BACKDROP', 'CURTAIN'):
      c, r = stack.pop(), stack.pop()
      at = cell(r, c, (world.rows, world.cols))
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
      at = cell(r, c, (world.rows, world.cols))
      if at is not None:
        me.curtain[at] = v != 0
    elif name == 'FILL':
      me.curtain[:] = stack.pop() != 0
    elif name == 'ANY':
      stack.append(int(ent(a).curtain.any()))
    elif name == 'MOVE':
      stack.append(0 if em.walker_move(me, world.board, plot, a) is None else 1)
    elif name == 'TELEPORT':
      c, r = stack.pop(), stack.pop()
      em.walker_teleport(me, r, c)
    elif name == 'REWARD':
      plot.add_reward(stack.pop())
    elif name == 'REWARD_F64':
      plot.add_reward(oc._f64(a, code[pc + 2]))
    elif name == 'TERMINATE':
      plot.terminate_episode(oc._f32(a))
    elif name == 'DISCOUNT':
      plot.discount = oc._f32(a)
    else:
      raise AssertionError('opcode %d' % op)
    pc = nxt
