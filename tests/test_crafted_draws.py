"""The draws the device restates, at MT19937 states crafted to reach their edges (no GPU):
tests/mt_states.py against CPython's `random` and NumPy's RandomState themselves; the
compiled-code oracle's draws (oracle/compiled.py) at rejection runs across the twist and at
every width edge; the float comparisons RANDCMP makes at the exact literal and one step
either side; and the Cued Catch boundary set, normal draws whose zz lies exactly on, or one
ulp either side of, -log(u2)."""

import operator

import numpy as np
import pytest

import mt_states as mts
from oracle import compiled as ocompiled
from pycolab_b200 import _lib

CHOSEN = [0x80000000, 0x5, 0x0, 0xffffffff, 0x7b]


@pytest.mark.parametrize('pos', [0, 1, 311, 622, 623, 624])
def test_crafted_outputs_come_out_of_both_generators(pos):
  words = mts.state(CHOSEN, pos, background=pos)
  r, rs = mts.python_random(words), mts.numpy_random(words)
  assert [r.getrandbits(32) for _ in CHOSEN] == CHOSEN
  assert [int(x) for x in rs.randint(0, 2 ** 32, size=len(CHOSEN), dtype=np.uint64)] == CHOSEN
  # on across one and then a second twist, word for word with the module's own MT19937
  rest = mts.outputs(words, len(CHOSEN) + 1300)[len(CHOSEN):]
  assert [r.getrandbits(32) for _ in rest] == rest
  assert [int(x) for x in rs.randint(0, 2 ** 32, size=len(rest), dtype=np.uint64)] == rest
  assert mts.python_words(r) == mts.numpy_words(rs)


def test_helpers_invert_and_encode():
  rs = np.random.RandomState(0)
  for y in [0, 1, 0xffffffff, 0x80000000] + [int(x) for x in rs.randint(0, 2 ** 32, 200,
                                                                         dtype=np.uint64)]:
    assert mts.temper(mts.untemper(y)) == y and mts.untemper(mts.temper(y)) == y
  words = mts.straddle([1, 2], [3, 4, 5], background=4)
  assert words[624] == 622 and mts.outputs(words, 5) == [1, 2, 3, 4, 5]
  assert all(words[:624]) and words[:5] == mts.state([], 624, background=4)[:5]
  for n in (0, 1, 2 ** 52, 2 ** 53 - 1, 3602879701896397):
    assert mts.python_random(mts.state(mts.split53(n), 0)).random() == n * 2.0 ** -53
  with pytest.raises(ValueError):
    mts.state([0] * 228, 620)                # 4 before the twist, and 223 after it at most
  r = mts.python_random(mts.state(mts.python_below(5, 2 ** 32), 623))
  assert r.getrandbits(33) == 5
  engine_row = mts.engine_row(type('G', (), {'rng_streams': ('python', 'numpy')}),
                              {'numpy': [1] * 625, 'python': [2] * 625})
  assert engine_row.dtype == np.uint32 and list(engine_row[::625]) == [2, 1]


# ------------------------------------------------------------ restated draws --

def _widths(python):
  w = [1, 2]
  for k in (1, 16, 31):
    w += [2 ** k, 2 ** k + 1]
  w.append(2 ** 32 - 1)
  if python:
    w.append(2 ** 32)
  return sorted(set(w))


def _run(n, python, rejections, accept):
  """Outputs for `rejections` rejected draws of width n, then one that gives `accept`, and
  the number of rejections (none where NumPy's mask is n - 1: it never rejects)."""
  below = mts.python_below if python else mts.numpy_below
  bad = 2 ** n.bit_length() - 1 if python else (1 << (n - 1).bit_length()) - 1
  if bad < n:
    rejections = 0
  return sum((below(bad, n) for _ in range(rejections)), []) + below(accept, n), rejections


# Rejection runs that cross the twist (half their outputs before it), and a long one from
# position 0.  Crafted outputs that cross the twist number at most 227 (mt_states.state), so
# the long run stays before it: 600 draws of one output, 300 of getrandbits(33)'s two.
RUNS = [1, 5, 110, 600]


@pytest.mark.parametrize('python', [False, True], ids=['numpy', 'python'])
@pytest.mark.parametrize('run', RUNS)
def test_restated_below_matches_the_generators(python, run):
  rejected = 0
  for n in _widths(python):
    words = 2 if python and n > 2 ** 32 - 1 else 1
    outs, rej = _run(n, python, run if run < 600 else 600 // words, n - 1 if n % 3 else n // 2)
    if n == 1 and not python:
      outs = []                                # randint(0, 1) consumes no output
    pos = 0 if run == 600 else 624 - len(outs) // 2
    words = mts.state(outs, pos, background=n % 1000)
    if python:
      r = mts.python_random(words)
      want = r.randrange(n)
      assert ocompiled.python_below(words, n) == want, (n, run)
      assert words == mts.python_words(r), (n, run)
    else:
      rs = mts.numpy_random(words)
      want = int(rs.randint(0, n))
      assert ocompiled.numpy_below(words, n) == want, (n, run)
      assert words == mts.numpy_words(rs), (n, run)
    assert want == (n - 1 if n % 3 else n // 2), (n, run)
    assert words[624] == (pos + len(outs)) % 624 or words[624] == pos + len(outs), (n, run)
    rejected += rej
  assert rejected >= 4 * run            # four widths of each generator reject


@pytest.mark.parametrize('pos', [0, 311, 622, 623, 624])
def test_restated_python_forms_match_random(pos):
  """randint, choice and random() through the restatement at crafted states: the whole
  int32 range (getrandbits(33), its first word at `pos`), one rejection then a value."""
  for low, high, rule, call in (
      (-2 ** 31, 2 ** 31 - 1, _lib.RAND_PYTHON_CLOSED, lambda r: r.randint(-2 ** 31, 2 ** 31 - 1)),
      (0, 5, _lib.RAND_PYTHON, lambda r: r.choice(range(5))),
      (-7, -2, _lib.RAND_PYTHON, lambda r: r.randrange(-7, -2))):
    n = high - low + (rule == _lib.RAND_PYTHON_CLOSED)
    outs = mts.python_below(2 ** n.bit_length() - 1, n) + mts.python_below(n - 1, n)
    words = mts.state(outs, pos, background=pos)
    r = mts.python_random(words)
    assert ocompiled.randint(words, rule, low, high) == call(r) == low + n - 1
    assert words == mts.python_words(r)
  words = mts.state(mts.split53(2 ** 52), pos)
  r, rs = mts.python_random(words), mts.numpy_random(words)
  x = ocompiled.random53(list(words))
  assert x == r.random() == rs.random_sample()


# ---------------------------------------------------------- RANDCMP's compare --

_OPS = {'EQ': operator.eq, 'NE': operator.ne, 'LT': operator.lt, 'LE': operator.le,
        'GT': operator.gt, 'GE': operator.ge}


@pytest.mark.parametrize('literal', [0.5, 0.25, 0.1])
def test_randcmp_at_the_literal_and_one_step_either_side(literal):
  """The draw RANDCMP makes (random53) at n = literal * 2^53 rounded down, and one step
  either side, compared with each operator: the oracle's table against Python's operator
  on CPython's own random()."""
  base = int(literal * 2 ** 53)
  seen = set()
  for n in (base - 1, base, base + 1):
    for pos in (0, 623):
      words = mts.state(mts.split53(n), pos, background=n & 0xff)
      x = ocompiled.random53(list(words))
      assert x == mts.python_random(words).random() == mts.numpy_random(words).random_sample()
      for name in ocompiled._CMP:
        for a, b in ((x, literal), (literal, x)):
          assert ocompiled._BINARY[name](a, b) == _OPS[name](a, b)
      seen.add((x > literal) - (x < literal))
  assert seen == ({-1, 0, 1} if literal != 0.1 else {-1, 1})


# ------------------------------------------------------ the Cued Catch boundary --

def test_cued_catch_boundary_set_decides_as_designed():
  cases, kept, dropped = mts.boundary_set()
  offsets = [c[2] for c in cases]
  assert dropped < 0.01 * (kept + dropped)
  for off in (-1, 0, 1):
    assert offsets.count(off) > 0.15 * kept, (off, offsets.count(off), kept)
  for m1, m2, offset in cases:
    words = mts.state(mts.pair_outputs(m1, m2), 0, background=m2 & 0xff)
    r = mts.python_random(words)
    r.normalvariate(0.0, 1.0)
    used = mts.python_words(r)[624]
    assert (used == 4) == (offset <= 0), (m1, m2, offset, used)
