"""Crafted MT19937 states: generators whose next outputs are chosen words, at any position and
across the twist.  No GPU.

A state is 625 words, the 624 key words and the position, as random.getstate()[1],
RandomState.get_state()[1:3] and each BatchedEngine rng slot hold it.  With position
p < 624 the next 624 - p outputs are temper(key[p..623]); the outputs after the twist are
new[i] = key[i + 397] ^ f(key[i], key[i + 1]) for i < 227, so key[i + 397] can be solved for
them as long as no output before the twist has fixed it.  Both random.setstate and
RandomState.set_state accept any such state, so the real generators are the ground truth at
every crafted edge.
"""

import decimal
import math

import numpy as np

N = 624
_UPPER, _LOWER, _MATRIX_A = 0x80000000, 0x7fffffff, 0x9908b0df


def temper(y):
  y ^= y >> 11
  y ^= (y << 7) & 0x9d2c5680
  y ^= (y << 15) & 0xefc60000
  return y ^ (y >> 18)


def _unshift_right(y, s):
  x = y
  for _ in range(32 // s + 1):
    x = y ^ (x >> s)
  return x


def _unshift_left(y, s, mask):
  x = y
  for _ in range(32 // s + 1):
    x = y ^ ((x << s) & mask)
  return x & 0xffffffff


def untemper(y):
  """The key word that `temper` turns into `y`."""
  y = _unshift_right(y, 18)
  y = _unshift_left(y, 15, 0xefc60000)
  y = _unshift_left(y, 7, 0x9d2c5680)
  return _unshift_right(y, 11)


def _f(a, b):
  y = (a & _UPPER) | (b & _LOWER)
  return (y >> 1) ^ (_MATRIX_A if y & 1 else 0)


def state(outputs, pos, background=0):
  """625 words whose next outputs, from position `pos` (0..624), are `outputs`.  Outputs past
  word 623 are the first ones after the twist; at most pos - 397 of them (227 from 624) can be
  chosen, since the words before the twist that they are solved into must be free.  Every
  other key word comes from RandomState(background)."""
  outputs = [int(x) & 0xffffffff for x in outputs]
  before, after = outputs[:N - pos], outputs[N - pos:]
  if after and len(after) > pos - 397:
    raise ValueError('%d outputs after the twist from position %d' % (len(after), pos))
  key = [int(w) for w in np.random.RandomState(background).get_state()[1]]
  for i, y in enumerate(before):
    key[pos + i] = untemper(y)
  for i, y in enumerate(after):
    key[397 + i] = untemper(y) ^ _f(key[i], key[i + 1])
  return key + [pos]


def straddle(before, after, background=0):
  """A state whose outputs `before` end at word 623 and `after` follow the twist."""
  return state(list(before) + list(after), N - len(before), background)


def outputs(words, n):
  """The next n outputs of `words` (left unchanged), by this module's own MT19937."""
  key, pos, out = list(words[:N]), int(words[N]), []
  for _ in range(n):
    if pos >= N:
      nxt = list(key)
      for j in range(N):
        nxt[j] = nxt[(j + 397) % N] ^ _f(nxt[j], nxt[(j + 1) % N])
      key, pos = nxt, 0
    out.append(temper(key[pos]))
    pos += 1
  return out


# ------------------------------------------------------------------ converters --

def python_state(words):
  """The argument of random.setstate."""
  return (3, tuple(int(w) for w in words), None)


def numpy_state(words):
  """The argument of RandomState.set_state."""
  return ('MT19937', np.array(words[:N], dtype=np.uint32), int(words[N]), 0, 0.0)


def python_random(words):
  import random
  r = random.Random()
  r.setstate(python_state(words))
  return r


def numpy_random(words):
  rs = np.random.RandomState()
  rs.set_state(numpy_state(words))
  return rs


def numpy_words(rs):
  _, key, pos = rs.get_state()[:3]
  return [int(w) for w in key] + [int(pos)]


def python_words(r):
  return [int(w) for w in r.getstate()[1]]


def engine_row(game, words):
  """One BatchedEngine rng_states row: `words[stream]` for each of game.rng_streams, in order."""
  return np.concatenate([np.asarray(words[s], dtype=np.uint32) for s in game.rng_streams])


# ------------------------------------------------------------------- encoders --

def split53(n):
  """The outputs a, b of which random() and random_sample() make n * 2^-53 (0 <= n < 2^53):
  (a >> 5) << 26 | b >> 6 == n.  The bits the draw drops are set."""
  assert 0 <= n < 2 ** 53
  return [(n >> 26) << 5 | 0x1f, (n & (2 ** 26 - 1)) << 6 | 0x3f]


def python_below(value, n):
  """The outputs of one getrandbits(n.bit_length()) in Random._randbelow(n) that give
  `value`: accepted when value < n, a rejection otherwise (value < 2^bit_length).  The bits
  getrandbits drops are set."""
  k = n.bit_length()
  assert 0 <= value < 2 ** k and k <= 33
  if k <= 32:
    return [value << (32 - k) | ((1 << (32 - k)) - 1)]
  return [value & 0xffffffff, (value >> 32) << 31 | _LOWER]


def numpy_below(value, n):
  """The output of which RandomState.randint(0, n) (masked rejection, 2 <= n <= 2^32) takes
  `value`: accepted when value < n, a rejection otherwise.  The bits above the mask are set."""
  mask = (1 << (n - 1).bit_length()) - 1
  assert 0 <= value <= mask
  return [(0xffffffff & ~mask) | value]


# ------------------------------------------------- Cued Catch's normal draws --
# random.normalvariate (Lib/random.py) accepts u1, u2 = random(), 1.0 - random() when
# zz = (NV_MAGICCONST * (u1 - 0.5) / u2) ** 2 / 4 <= -log(u2).

NV_MAGICCONST = 4 * math.exp(-0.5) / math.sqrt(2.0)


def _zz(m1, u2):
  u1 = m1 * 2.0 ** -53
  z = NV_MAGICCONST * (u1 - 0.5) / u2
  return z * z / 4.0


def _first_m1(target, u2):
  """The least 53-bit m1 >= 2^52 with _zz(m1, u2) >= target (zz rises with m1 there)."""
  lo, hi = 2 ** 52, 2 ** 53 - 1
  if _zz(hi, u2) < target:
    return None
  while lo < hi:
    mid = (lo + hi) // 2
    if _zz(mid, u2) >= target:
      hi = mid
    else:
      lo = mid + 1
  return lo


def correctly_rounded_log(u2):
  with decimal.localcontext() as ctx:
    ctx.prec = 60
    return float(decimal.Decimal(u2).ln())


def boundary_set(count=1893, seed=2024):
  """[(m1, m2, offset)]: random() draws m1 * 2^-53 and m2 * 2^-53 making normalvariate's
  u1 and u2 = 1 - m2 * 2^-53 in [0.05, 1), with zz exactly -log(u2) moved by `offset` ulps
  (-1, 0, +1).  Only u2 whose math.log is correctly rounded (60 decimal digits) are kept;
  returns (cases, kept, dropped)."""
  rs = np.random.RandomState(seed)
  cases, dropped = [], 0
  for m2 in rs.randint(1, int(0.95 * 2 ** 53), size=count, dtype=np.int64):
    u2 = 1.0 - int(m2) * 2.0 ** -53
    if math.log(u2) != correctly_rounded_log(u2):
      dropped += 1
      continue
    t = -math.log(u2)
    for offset, target in ((-1, math.nextafter(t, 0.0)), (0, t), (1, math.nextafter(t, math.inf))):
      m1 = _first_m1(target, u2)
      if m1 is not None and _zz(m1, u2) == target:
        cases.append((m1, int(m2), offset))
  return cases, count - dropped, dropped


def pair_outputs(m1, m2):
  """The four outputs of normalvariate's random() draws m1 * 2^-53 and m2 * 2^-53."""
  return split53(m1) + split53(m2)
