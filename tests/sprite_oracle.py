"""CPU interpreter of compiled games with plain Sprites (include/pcl.h PCL_OP_SETFIELD,
pcl_spec.program_arg[3]).  TEST INFRASTRUCTURE ONLY.

Every opcode but SETFIELD is interpreted by tests/scrolling_oracle.py, unchanged.  This
module builds its world and hands it a copy of the code in which each `SETFIELD f` is a
`SETR` of a register slot past a plain Sprite's five (SETFIELD_SLOT + f): both pop one value
and take one operand word, so every address stays where it was.  A plain Sprite's register
list sends those slots to the sprite's row, column or visibility; its other slots are its
registers VROW, VCOL and AUX0-AUX2, in that order.

A plain Sprite is an engine_model walker whose row, col and visible SETFIELD sets.
engine_model's render paints it with NumPy indexing, `board[row, col]`: a negative index
counts from the end once, and a visible sprite still off the board raises IndexError, as
upstream's render does (rendering.py:139).  The device latches PCL_ENV_ERR_INDEX there.
"""

import scrolling_oracle
from pycolab_b200 import _lib

SETFIELD_SLOT = 100             # SETFIELD f runs as SETR (SETFIELD_SLOT + f)


class PlainRegisters(list):
  """A plain Sprite's registers; slots SETFIELD_SLOT + f write its row, col or visible."""

  def __init__(self, sprite, words):
    super(PlainRegisters, self).__init__(words)
    self.sprite = sprite

  def __setitem__(self, i, v):
    if isinstance(i, int) and i >= SETFIELD_SLOT:
      f = i - SETFIELD_SLOT
      if f == _lib.FIELD_VISIBLE:
        self.sprite.visible = v != 0
      else:
        setattr(self.sprite, 'row' if f == _lib.FIELD_ROW else 'col', v)
    else:
      super(PlainRegisters, self).__setitem__(i, v)


def _without_setfield(code):
  """`code` with each SETFIELD f as SETR (SETFIELD_SLOT + f)."""
  out = list(code)
  n = code[0]
  pc = 1 + n
  while pc < len(code):
    op = code[pc]
    if op == _lib.OP['SETFIELD']:
      out[pc], out[pc + 1] = _lib.OP['SETR'], SETFIELD_SLOT + code[pc + 1]
    pc += 1 + _lib.OPERANDS[op] + (code[pc + 1] if op in (_lib.OP['IN'], _lib.OP['PICK']) else 0)
  return out


def make_world(game, words=None):
  """A fresh oracle env (the its_showtime() state) of lowered compiled game `game`, its plain
  Sprites included.  `words`: as oracle.compiled.make_world."""
  world = scrolling_oracle.make_world(game, words)
  for s, ch in enumerate(game.sprite_chars):
    if (game.program_arg[3] >> s) & 1:
      rec = game.sprites[s]
      w = world.things[ch]
      w.regs = PlainRegisters(w, [int(x) for x in list(rec[_lib.S_VROW:_lib.S_VCOL + 1]) +
                                  list(rec[_lib.S_AUX0:])])
  world.code = _without_setfield(world.code)
  return world
