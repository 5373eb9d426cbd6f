"""Device draws against CPython's `random` and NumPy's RandomState at crafted generator states
(tests/mt_states.py): every env of one BatchedEngine starts from its own state, so positions
at and around the twist, rejection runs that cross it and draws exactly on a decision
boundary run side by side in one launch.  Each case steps the engine in lock-step with
oracle worlds whose real generators start from the same states, through auto-resets, and
ends by comparing every env's generator words."""

import random

import numpy as np
import pytest

import mt_states as mts
import registered_games as rg
from registered_games import global_generators  # noqa: F401  (a fixture)
from oracle import compiled as ocompiled
from oracle import cued_catch as occ
from oracle import games as ogames
from oracle import sampled_check
from oracle import sequence_recall as osr
from oracle import t_maze as otm
from pycolab_b200 import _lib, lowering

pytestmark = pytest.mark.gpu

ACCEPT = 0x00000003      # below any width of 4 or more, in mt_below and _randbelow alike


def _engine(games, rows, **kw):
  from pycolab_b200 import batched
  eng = batched.BatchedEngine(games, batch=len(rows), rng_states=np.stack(rows), **kw)
  eng.its_showtime()
  return eng


def _words(eng):
  """u32 [B, slots, 625]: every env's generator words now."""
  return eng.rng.cpu().numpy().view(np.uint32).reshape(eng.batch, -1, _lib.MT_WORDS)


def _actions(seed, T, B, choices, p=None):
  rs = np.random.RandomState(seed)
  return np.stack([rs.choice(choices, size=B, p=p) for _ in range(T)]).astype(np.int32)


def _fill(pos, make, background):
  """A state at `pos` holding as many of make(k), k = 0, 1, ... (lists of outputs) as fit."""
  room = 624 - pos + max(0, pos - 397) if pos < 624 else 227
  outs, k = [], 0
  while len(outs) + len(make(k)) <= room:
    outs += make(k)
    k += 1
  return mts.state(outs, pos, background), k


def _runs(background):
  """0xffffffff runs (rejected by every width that is not a power of two) and then ACCEPT:
  short and long runs across the twist, and one of 600 from position 0."""
  out = []
  for run, pos in ((1, 623), (5, 622), (100, 570), (225, 520), (600, 0), (0, 623), (0, 624)):
    out.append(mts.state([0xffffffff] * run + [ACCEPT], pos, background + run))
  return out


# ----------------------------------------------------------------- apprehend --

def test_apprehend_uniform_at_every_edge():
  """The restart's random.uniform from r53 in {0, 2^-53, 0.5, 1 - 2^-53}, its two words at
  positions 0, 1, 2, 311, 622, 623 (straddling the twist) and 624."""
  from pycolab_b200.games import apprehend
  art = apprehend.GAME_ART
  game = lowering.lower(apprehend.make_game(art))
  states = [mts.state(mts.split53(n), pos, background=k)
            for k, (pos, n) in enumerate((pos, n) for pos in (0, 1, 2, 311, 622, 623, 624)
                                         for n in (0, 1, 2 ** 52, 2 ** 53 - 1))]
  rngs = [mts.python_random(w) for w in states]
  eng = _engine([game], [mts.engine_row(game, {'python': w}) for w in states])

  def same_dx(t, eng, worlds, outs):
    spr = eng.sprites.cpu().numpy()
    for e, w in worlds.items():
      dx = np.array(spr[e, 1, _lib.S_AUX0:_lib.S_AUX0 + 2], dtype='<i4').view('<f8')[0]
      assert dx == w.things['b'].aux['dx'], (t, e)
  sampled_check.lockstep(eng, lambda e: ogames.make_apprehend(art, rngs[e]), range(len(states)),
                         _actions(3, 100, len(states), [0, 1, 2]), on_step=same_dx)
  words = _words(eng)
  for e, r in enumerate(rngs):
    assert words[e, 0].tolist() == mts.python_words(r), e


# -------------------------------------------------------------------- t_maze --

SPECKLE = (3602879701896396, 3602879701896397)    # below 0.4 = 3602879701896397 * 2^-53, and not


def _t_maze_states():
  """(python, numpy) word pairs: the cue's random() at 0.5 and one step below it, across the
  twist and not; the speckle's NumPy stream at odd and even positions, its first pairs
  alternating on either side of 0.4 (at position 623 the first pair, either value, is split
  by the twist)."""
  cues = [mts.state(mts.split53(n), pos, background=pos)
          for pos in (0, 311, 623) for n in (2 ** 52, 2 ** 52 - 1)]
  speckles = [_fill(pos, lambda k: mts.split53(SPECKLE[(k + shift) % 2]), 100 + pos)[0]
              for pos, shift in ((1, 0), (3, 0), (311, 0), (623, 0), (623, 1), (0, 0), (622, 0),
                                 (624, 0))]
  return [(c, s) for c in cues for s in speckles]


def test_t_maze_cue_and_speckle_at_every_edge():
  from pycolab_b200 import levels
  from pycolab_b200.games import t_maze
  cfg = (0, False, 25, 0, 0)
  maze, cue = levels.t_maze_level(0)
  # Speckle in the first two pattern rows, far from the player, where the crafted draws land.
  maze = ['*' * len(maze[0])] * 2 + list(maze[2:])
  game = lowering.lower(t_maze.make_game(*cfg, maze_art=maze, cue_art=cue))
  pairs = _t_maze_states()
  rngs = {e: (mts.python_random(p), mts.numpy_random(n)) for e, (p, n) in enumerate(pairs)}
  eng = _engine([game], [mts.engine_row(game, {'python': p, 'numpy': n}) for p, n in pairs])
  dirt = game.drape_chars.index('*')
  cues = set()

  def whole_speckle(t, eng, worlds, outs):
    if t:
      return
    pattern = eng.patterns[dirt].cpu().numpy().view(np.uint32).reshape(eng.batch,
                                                                        game.pattern_rows, -1)
    for e, w in worlds.items():
      got = lowering.unpack_rows(pattern[e], game.pattern_cols)
      np.testing.assert_array_equal(got, w.things['*'].pattern, err_msg=str(e))
      cues.add(w.things['Q'].aux['which_goal'])
  sampled_check.lockstep(eng, lambda e: otm.make_t_maze(maze, cue, *cfg, rng=rngs[e][0],
                                                        np_rng=rngs[e][1]),
                         range(len(pairs)), _actions(5, 60, len(pairs), [1, 2, 3, 4, 5]),
                         curtains='*', on_step=whole_speckle)
  assert cues == {'left', 'right'}
  words = _words(eng)
  for e, (r, rs) in rngs.items():
    assert words[e, 0].tolist() == mts.python_words(r), e
    assert words[e, 1].tolist() == mts.numpy_words(rs), e


# ------------------------------------------------------- marauders, shockwave --

def test_marauders_choice_rejects_across_the_twist():
  from pycolab_b200 import levels
  from pycolab_b200.games import extraterrestrial_marauders as g
  art = levels.marauders_level()
  game = lowering.lower(g.make_game(art))
  states = _runs(0) * 2
  rngs = [mts.numpy_random(w) for w in states]
  eng = _engine([game], [mts.engine_row(game, {'numpy': w}) for w in states])
  sampled_check.lockstep(eng, lambda e: ogames.make_marauders(art, rngs[e]), range(len(states)),
                         _actions(7, 200, len(states), [0, 1, 2, 3]))
  words = _words(eng)
  for e, rs in enumerate(rngs):
    assert words[e, 0].tolist() == mts.numpy_words(rs), e
    assert mts.numpy_words(rs) != states[e], e             # every env drew


@pytest.mark.parametrize('shape', [(32, 64), (5, 13)], ids=['2048_cells', '65_cells'])
def test_shockwave_randint_rejects_across_the_twist(shape):
  """H * W a power of two (mt_below never rejects) and 65 (almost half of all draws do)."""
  from pycolab_b200 import levels
  from pycolab_b200.games import shockwave
  arts = [levels.shockwave_level(30 + i, shape[0], shape[1], 0.45) for i in range(2)]
  games = [lowering.lower(shockwave.make_game(a)) for a in arts]
  states = _runs(1) * 2
  rngs = [mts.numpy_random(w) for w in states]
  eng = _engine(games, [mts.engine_row(games[0], {'numpy': w}) for w in states])
  sampled_check.lockstep(eng, lambda e: ogames.make_shockwave(arts[e % 2], rngs[e]),
                         range(len(states)), _actions(4, 120, len(states), [0, 1, 2, 3, 4],
                                                      p=[.6, .12, .12, .12, .04]),
                         curtains='@')
  words = _words(eng)
  for e, rs in enumerate(rngs):
    assert words[e, 0].tolist() == mts.numpy_words(rs), e


# ----------------------------------------------------------- sequence_recall --

def _sequence_outputs(k):
  """Light k of the sequence: k % 3 rejections (getrandbits(3) >= 4), then light k % 4."""
  return sum((mts.python_below(4 + (k + j) % 4, 4) for j in range(k % 3)), []) + \
      mts.python_below(k % 4, 4)


def test_sequence_recall_lights_drawn_across_the_twist():
  from pycolab_b200 import levels
  from pycolab_b200.games import sequence_recall
  args = (16, 1, 1, 1, 200)
  art = levels.sequence_recall_art(9, 13)
  random.seed(0)
  game = lowering.lower(sequence_recall.make_game(*args, art=art))
  seq = sum((_sequence_outputs(k) for k in range(16)), [])
  states = [mts.state(seq, pos, background=pos) for pos in (624 - len(seq) // 2, 600, 623, 0, 624)]
  rngs = [mts.python_random(w) for w in states]
  eng = _engine([game], [mts.engine_row(game, {'python': w}) for w in states])
  sampled_check.lockstep(eng, lambda e: osr.make_sequence_recall(art, *args, rng=rngs[e]),
                         range(len(states)),
                         _actions(3, 300, len(states), [1, 2, 3, 4, 5, 0, 6],
                                  p=[.24, .24, .24, .24, .02, .01, .01]),
                         curtains='M%', sprites='P')
  words = _words(eng)
  for e, r in enumerate(rngs):
    assert words[e, 0].tolist() == mts.python_words(r), e


# ---------------------------------------------------------------- cued_catch --

NOISY = (1, 1, 10 ** 6, False, 1.25, 0)           # every frame in the ball column pays noise


class _Spy(random.Random):
  """A Random that notes its position when normalvariate is first called."""
  first = None

  def normalvariate(self, mu=0.0, sigma=1.0):
    if self.first is None:
      self.first = self.getstate()[1][624]
    return super(_Spy, self).normalvariate(mu, sigma)


def _first_normal(art, args, words, frames=None):
  """The position the first normalvariate of a world from `words` starts at.  With `frames`
  (a list), the frame it is drawn in is appended to it."""
  spy = _Spy()
  spy.setstate(mts.python_state(words))
  w = occ.make_cued_catch(art, *args, rng=spy)
  w.its_showtime()
  frame = 0
  while spy.first is None:
    w.play(3)
    frame += 1
  if frames is not None:
    frames.append(frame)
  return spy.first


def _pairing_outputs(k):
  """_randbelow(4 - k) of random.sample's pool: one or two rejections, then a value."""
  n = 4 - k
  bad = 2 ** n.bit_length() - 1
  return mts.python_below(bad, n) * (1 + k % 2) + mts.python_below(k % n, n)


def test_cued_catch_pairings_and_random_across_the_twist():
  """random.sample's _randbelow(4), (3), (2), (1) after rejections (_randbelow(1) rejects
  whenever the top bit is set), across the twist; and normalvariate's first random()
  with its two words straddling it."""
  from pycolab_b200 import levels
  from pycolab_b200.games import cued_catch
  args = (2, 3, 4, False, 0.0, 0)
  art = levels.cued_catch_art()
  pool = sum((_pairing_outputs(k) for k in range(4)), [])
  states = [mts.state(pool, pos, background=pos) for pos in (624 - len(pool) // 2, 623, 0, 624)]
  noisy_art = levels.cued_catch_art(7, 12, player=(1, 3), balls=((1, 3), (1, 3)))
  straddles = []
  for start in range(623 - len(pool), 400, -1):      # the first u1's words at 623 and 0
    words = mts.state(pool, start, background=start)
    if _first_normal(noisy_art, NOISY, words) == 623:
      straddles.append(words)
  assert straddles
  random.seed(0)
  for a, rows in ((art, args), (noisy_art, NOISY)):
    game = lowering.lower(cued_catch.make_game(*rows, art=a))
    cases = states if a is art else straddles[:4]
    rngs = [mts.python_random(w) for w in cases]
    eng = _engine([game], [mts.engine_row(game, {'python': w}) for w in cases])
    sampled_check.lockstep(eng, lambda e: occ.make_cued_catch(a, *rows, rng=rngs[e]),
                           range(len(cases)), _actions(9, 120, len(cases), [1, 2, 3]))
    words = _words(eng)
    for e, r in enumerate(rngs):
      assert words[e, 0].tolist() == mts.python_words(r), e


def test_cued_catch_normal_draws_on_the_accept_boundary():
  """Every case of the boundary set, one per env: zz exactly -log(u2), and one ulp either
  side, placed where the env's first normalvariate takes its u1.  The paid reward's float64
  bits and the words left behind show whether the pair was accepted."""
  from pycolab_b200 import levels
  from pycolab_b200.games import cued_catch
  cases, _, _ = mts.boundary_set(5600)
  B = len(cases)
  assert B >= 4096
  art = levels.cued_catch_art(7, 12, player=(1, 3), balls=((1, 3), (1, 3)))
  states, frames = [], []
  for e, (m1, m2, _) in enumerate(cases):
    background = mts.state([], 0, background=e)
    at = _first_normal(art, NOISY, background, frames)
    states.append(mts.state(mts.outputs(background, at) + mts.pair_outputs(m1, m2), 0,
                            background=e))
  random.seed(0)
  game = lowering.lower(cued_catch.make_game(*NOISY, art=art))
  rngs = [mts.python_random(w) for w in states]
  eng = _engine([game], [mts.engine_row(game, {'python': w}) for w in states])
  sampled_check.lockstep(eng, lambda e: occ.make_cued_catch(art, *NOISY, rng=rngs[e]), range(B),
                         np.full((max(frames) + 1, B), 3, np.int32))
  words = _words(eng)
  for e, r in enumerate(rngs):
    assert words[e, 0].tolist() == mts.python_words(r), e


# ------------------------------------------------------------------ compiled --

@pytest.fixture(scope='module')
def games():
  yield from rg.registered('drawn_games.py')


def _compiled_lockstep(lowered, word_sets, T, n_actions, seed):
  """word_sets[e]: {stream: words}; the oracle's worlds draw from copies of them."""
  eng = _engine([lowered], [mts.engine_row(lowered, w) for w in word_sets])
  words = {e: [list(w[s]) for s in lowered.rng_streams] for e, w in enumerate(word_sets)}
  sampled_check.lockstep(eng, lambda e: ocompiled.make_world(lowered, words[e]),
                         range(len(word_sets)), _actions(seed, T, len(word_sets),
                                                         list(range(n_actions))),
                         pad_columns=True, on_step=rg.register_check(lambda e: lowered))
  got = _words(eng)
  for e in words:
    assert got[e].tolist() == words[e], e
  return eng


def test_monsters_draws_straddle_the_twist(games):
  """Both generators start at every position from 560 to 624, against each other, so each
  draw kind (random(), rand(), choice, randint of either generator) meets the twist."""
  lowered = lowering.lower(games.make_monsters(0))
  sets = [{'numpy': mts.state([], 560 + k, background=k),
           'python': mts.state([], 624 - k, background=100 + k)} for k in range(65)]
  _compiled_lockstep(lowered, sets, 60, games.N_ACTIONS['monsters'], 11)


def test_getrandbits_33_at_word_623(games):
  """Edges' random.randint(-2^31, 2^31 - 1): the two-word getrandbits(33) from word 623,
  rejected once across the twist, then accepted."""
  from pycolab_b200 import compiler
  lowered = lowering.lower(games.make_edges(0))
  slot = compiler.registered(games.Edges).slot('case')
  py = lowered.rng_streams.index('python')
  # Python draws at cases 2, 4, ... 12 of widths 1, 3, 2^16 + 1, 2^30 + 1, 2^31 and 2^31 + 1
  # (value 0 each), then case 14: one rejection and an accepted value, from word 623 on.
  outs = sum((mts.python_below(0, n) for n in (1, 3, 2 ** 16 + 1, 2 ** 30 + 1, 2 ** 31,
                                                2 ** 31 + 1)), [])
  outs += mts.python_below(2 ** 33 - 1, 2 ** 32) + mts.python_below(5, 2 ** 32)
  sets = []
  for k in range(4):
    w = {'numpy': mts.state([], 624 - k, background=k), 'python': mts.state(outs, 617, k)}
    world = ocompiled.make_world(lowered, [list(w[s]) for s in lowered.rng_streams])
    world.its_showtime()
    while world.things['x'].regs[slot] != 14:
      world.play(0)
    assert world.rng[py][624] == 623
    sets.append(w)
  assert sets
  _compiled_lockstep(lowered, sets, 40, 2, 12)


def test_thresholds_on_and_beside_each_literal(games):
  """Every float draw of Thresholds at n = literal * 2^53 and one step either side, from
  crafted words straddling the twist and not, in both generators."""
  lowered = lowering.lower(games.make_thresholds(0))
  lit = games.THRESHOLDS

  def draw(shift):
    return lambda k: mts.split53(int(lit[k % 12] * 2 ** 53) + (k + shift) % 3 - 1)
  sets = []
  for k, (pn, pp) in enumerate(((0, 0), (623, 624), (624, 623), (311, 601), (601, 311))):
    for shift in range(3):
      sets.append({'numpy': _fill(pn, draw(shift), k)[0],
                   'python': _fill(pp, draw(shift + 1), 50 + k)[0]})
  _compiled_lockstep(lowered, sets, 12, 1, 13)


# -------------------------------------------------------------------- facade --

@pytest.mark.parametrize('pos', [1, 623])
def test_facade_continues_the_global_generators(games, global_generators, pos):  # noqa: F811
  """A marauders Engine and a drawn-games Engine, the global generators left at `pos`: after
  every step they hold the oracle's generators' words."""
  from pycolab_b200 import levels
  from pycolab_b200.games import extraterrestrial_marauders as g
  art = levels.marauders_level()
  np.random.set_state(mts.numpy_state(mts.state([], pos, background=pos)))
  rs = mts.numpy_random(mts.state([], pos, background=pos))
  engine, world = g.make_game(art), ogames.make_marauders(art, rs)
  engine.its_showtime()
  world.its_showtime()
  acts = _actions(2, 150, 1, [0, 1, 2, 3])[:, 0]
  for t, a in enumerate(acts):
    if world.game_over:
      break
    board, _, _ = engine.play(int(a))
    want = world.play(int(a))
    assert np.array_equal(board.board if hasattr(board, 'board') else board, want[0]), t
    assert rg.global_words('numpy') == mts.numpy_words(rs), t

  lowered = lowering.lower(games.make_monsters(1))
  words = {s: mts.state([], pos, background=pos + k) for k, s in enumerate(lowered.rng_streams)}
  random.setstate(mts.python_state(words['python']))
  np.random.set_state(mts.numpy_state(words['numpy']))
  engine = games.make_monsters(1)
  world = ocompiled.make_world(lowered, [list(words[s]) for s in lowered.rng_streams])
  engine.its_showtime()
  world.its_showtime()
  for t, a in enumerate(_actions(3, 80, 1, [0, 1, 2, 3, 4])[:, 0]):
    if world.game_over:
      break
    engine.play(int(a))
    world.play(int(a))
    for k, s in enumerate(lowered.rng_streams):
      assert rg.global_words(s) == world.rng[k], (t, s)
