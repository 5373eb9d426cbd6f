"""CPU interpreter of compiled games whose Backdrop has update() code (include/pcl.h
PCL_OP_SETBACK / FILLBACK / ROLLBACK, pcl_spec.program_arg[4]).  TEST INFRASTRUCTURE ONLY.

The world is tests/sprite_oracle.py's, and its entities run there.  This module
adds the Backdrop: engine_model runs `world.backdrop_program` before update group 0 on the
board of the last render (engine.py:718-723), and every render paints `world.backdrop`, which
the function below writes.  Its code is the function whose entry is header word 1 + n; a
Backdrop function has no registers and no entity of its own, so only the opcodes
pcl_bind_code accepts there are interpreted.  The three Backdrop opcodes are restated from
NumPy: a cell write, a fill, and np.roll of a band of rows.
"""

import numpy as np

import scrolling_oracle
import sprite_oracle
from oracle import compiled as oc
from oracle import engine_model as em
from pycolab_b200 import _lib

_ERR_INDEX, _ERR_ARITH, _ERR_RANGE = 0x8, 0x20, 0x40
_BINARY = {'ADD': lambda x, y: x + y, 'SUB': lambda x, y: x - y, 'MUL': lambda x, y: x * y,
           'FLOORDIV': lambda x, y: x // y, 'MOD': lambda x, y: x % y,
           'EQ': lambda x, y: x == y, 'NE': lambda x, y: x != y, 'LT': lambda x, y: x < y,
           'LE': lambda x, y: x <= y, 'GT': lambda x, y: x > y, 'GE': lambda x, y: x >= y}
_CMP = ('EQ', 'NE', 'LT', 'LE', 'GT', 'GE')


def make_world(game, words=None):
  """A fresh oracle env (the its_showtime() state) of lowered compiled game `game`, its
  Backdrop's code included.  `words`: as oracle.compiled.make_world."""
  if not game.program_arg[4]:
    return sprite_oracle.make_world(game, words)
  # sprite_oracle's world, built as its make_world builds it; the code header has one word
  # more (the Backdrop's entry), so the SETFIELD rewrite walks the functions from 2 + n.
  world = scrolling_oracle.make_world(game, words)
  for s, ch in enumerate(game.sprite_chars):
    if (game.program_arg[3] >> s) & 1:
      rec = game.sprites[s]
      w = world.things[ch]
      w.regs = sprite_oracle.PlainRegisters(w, [int(x) for x in list(rec[_lib.S_VROW:_lib.S_VCOL + 1]) +
                                                list(rec[_lib.S_AUX0:])])
  code = list(world.code)
  pc = 2 + code[0]
  while pc < len(code):
    op = code[pc]
    if op == _lib.OP['SETFIELD']:
      code[pc], code[pc + 1] = _lib.OP['SETR'], sprite_oracle.SETFIELD_SLOT + code[pc + 1]
    pc += 1 + _lib.OPERANDS[op] + (code[pc + 1] if op in (_lib.OP['IN'], _lib.OP['PICK']) else 0)
  world.code = code
  world.backdrop_program = backdrop_program
  return world


def backdrop_program(world, actions):
  """The Backdrop's update(): its compiled words, one instruction at a time."""
  code, plot = world.code, world.plot
  chars = world.entity_chars
  bd = world.backdrop
  action = _lib.ACTION_NONE if actions is None else int(actions)
  stack, local = [], [0] * _lib.CODE_LOCALS
  pc = code[1 + len(chars)]

  def cell(r, c):
    r = r + world.rows if r < 0 else r
    c = c + world.cols if c < 0 else c
    if 0 <= r < world.rows and 0 <= c < world.cols:
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
    elif name == 'SETBACK':
      v, c, r = stack.pop(), stack.pop(), stack.pop()
      at = cell(r, c)
      if at is not None:
        bd[at] = v & 0xff
    elif name == 'FILLBACK':
      bd[:] = stack.pop() & 0xff
    elif name == 'ROLLBACK':
      lo, hi = code[pc + 2], code[pc + 3]
      bd[lo:hi] = np.roll(bd[lo:hi], stack.pop(), axis=a)
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
      w = world.things[chars[a]]
      stack.append((w.row, w.col, w.vrow, w.vcol, int(bool(w.visible)))[code[pc + 2]])
    elif name == 'GETP':
      stack.append(plot.regs[a])
    elif name == 'SETP':
      plot.regs[a] = stack.pop()
    elif name in ('BOARD', 'BACKDROP', 'CURTAIN'):
      c, r = stack.pop(), stack.pop()
      at = cell(r, c)
      if at is None:
        stack.append(0)
      elif name == 'BOARD':
        stack.append(int(world.board[at]))
      elif name == 'BACKDROP':
        stack.append(int(bd[at]))
      else:
        stack.append(int(world.things[chars[a]].curtain[at]))
    elif name == 'ANY':
      stack.append(int(world.things[chars[a]].curtain.any()))
    elif name == 'PATTERN':
      c, r = stack.pop(), stack.pop()
      pattern = world.things[chars[a]].pattern
      r, c = r + pattern.shape[0] if r < 0 else r, c + pattern.shape[1] if c < 0 else c
      if 0 <= r < pattern.shape[0] and 0 <= c < pattern.shape[1]:
        stack.append(int(pattern[r, c]))
      else:
        world.error |= _ERR_INDEX
        stack.append(0)
    elif name == 'PATANY':
      stack.append(int(world.things[chars[a]].pattern.any()))
    elif name in ('PRESCROLL', 'POSTSCROLL'):
      c, r = stack.pop(), stack.pop()
      fn = em.scrolly_prescroll if name == 'PRESCROLL' else em.scrolly_postscroll
      stack.extend(oc._wrap32(x) for x in fn(world.things[chars[a]], (r, c), plot))
    elif name == 'REWARD':
      plot.add_reward(stack.pop())
    elif name == 'REWARD_F64':
      plot.add_reward(oc._f64(a, code[pc + 2]))
    elif name == 'TERMINATE':
      plot.terminate_episode(oc._f32(a))
    elif name == 'DISCOUNT':
      plot.discount = oc._f32(a)
    else:
      raise AssertionError('opcode %s in a Backdrop function' % name)
    pc = nxt
