"""Seeded resets on the H100: `pcl_seed_rng` and `BatchedEngine.reset(mask, seeds=)`.

- Words: every seeded (env, slot) holds `_mt_state`'s words, through every slot kind and both
  slots of two-slot handles; guard words around the rows, and unmasked envs' words, records
  and outputs, stay byte for byte.
- Reference parity: an engine built with another rng_seed, reset(mask, seeds=golden seed),
  replays every golden that records a seed, several goldens of one art per engine beside
  distractor envs, through auto-restarts.
- An engine built with rng_seed=a equals one built with b and reset(seeds=a).
- The constructor's kernel-seeded words equal the host loop's; a shard's env_offset too.
- A captured reset(mask, seeds) + 100 steps replays a changed seed tensor as an eager twin.
- A seeded reset restarts the time-limit count and the episode return, as a masked one does.
"""

import json

import numpy as np
import pytest
import torch

import example_games as eg
import golden_cases as gc
import registered_games as rg
from registered_games import global_generators  # noqa: F401  (a fixture)
from pycolab_b200 import _lib, batched, levels, lowering

pytestmark = pytest.mark.gpu

DISTRACTORS = 2
MIXED = [0, 1, 2 ** 31 - 1, 2 ** 31, 2 ** 32 - 1]


def _sync():
  torch.cuda.synchronize()


def _t_maze():
  from pycolab_b200.games import t_maze
  return t_maze.make_game(1, False, limbo_time=3)


def _makers():
  """{name: make() -> facade Engine} of a level of every program with generator slots."""
  from pycolab_b200.games import apprehend, cued_catch, sequence_recall, shockwave
  from pycolab_b200.games import extraterrestrial_marauders as marauders
  return {
      'marauders': lambda: marauders.make_game(levels.marauders_level()),
      'shockwave': lambda: shockwave.make_game(0),
      'apprehend': apprehend.make_game,
      'cued_catch': lambda: cued_catch.make_game(2, 2, 4),
      'sequence_recall': lambda: sequence_recall.make_game(2, 3, 2, 2),
      't_maze': _t_maze,
  }


PROGRAMS = sorted(_makers()) + ['compiled']


@pytest.fixture(scope='module')
def drawn():
  yield from rg.registered('drawn_games.py')


def _game(name, drawn):
  return lowering.lower(drawn.make_monsters(0) if name == 'compiled' else _makers()[name]())


def _words(eng):
  return eng.rng.cpu().numpy().view(np.uint32).reshape(eng.batch, -1, _lib.MT_WORDS)


def _host_words(game, seeds):
  return np.stack([np.stack([batched._mt_state(s, int(seed)) for s in game.rng_streams])
                   for seed in seeds])


def _records(eng):
  out = [eng.sprites, eng.drapes, eng.plot, eng._board, eng.reward, eng.has_reward,
         eng.discount, eng.done]
  return [t.cpu().clone() for t in out]


# ---- words ------------------------------------------------------------------------------

@pytest.mark.parametrize('name', ['t_maze', 'compiled', 'apprehend', 'marauders'])
def test_seeded_words_are_the_hosts(global_generators, drawn, name):  # noqa: F811
  game = _game(name, drawn)
  B, G = 4099, 1000
  eng = batched.BatchedEngine([game], batch=B, rng_seed=77)
  eng.its_showtime()
  slots = len(game.rng_streams)
  # the rows inside guard words on both sides
  guarded = torch.full((B * slots * _lib.MT_WORDS + 2 * G,), 0x5a5a5a5a, dtype=torch.int32,
                       device=eng.device)
  guarded[G:-G].copy_(eng.rng.reshape(-1))
  eng.rng = guarded[G:-G].view(B, slots * _lib.MT_WORDS)
  eng._state.d_rng = eng.rng.data_ptr()
  _lib.check(eng._lib.pcl_bind_state(eng._h, batched.C.byref(eng._state)), 'pcl_bind_state')
  rs = np.random.RandomState(5)
  seeds = np.array([MIXED[e] if e < len(MIXED) else int(rs.randint(0, 2 ** 32, dtype=np.int64))
                    for e in range(B)], dtype=np.int64)
  mask = rs.rand(B) < 0.6
  mask[:len(MIXED)] = True
  mask[-1] = False
  before_words, before = _words(eng).copy(), _records(eng)
  d_mask = torch.from_numpy(mask.astype(np.uint8)).cuda()
  eng._seed(d_mask, eng._seed_tensor(seeds))
  _sync()
  got = _words(eng)
  want = _host_words(game, seeds[mask])
  assert np.array_equal(got[mask], want)
  assert np.array_equal(got[~mask], before_words[~mask])
  for a, b in zip(before, _records(eng)):      # nothing but d_rng is written
    assert torch.equal(a, b)
  g = guarded.cpu()
  assert bool((g[:G] == 0x5a5a5a5a).all()) and bool((g[-G:] == 0x5a5a5a5a).all())
  # NULL mask: every env
  eng._seed(None, eng._seed_tensor(3))
  _sync()
  assert np.array_equal(_words(eng), _host_words(game, np.arange(3, 3 + B)))


# ---- reference parity -------------------------------------------------------------------

def _family_goldens():
  """[(family, [golden names])] of every FAMILIES golden that records a seed, grouped by
  everything their engine is built from but the seed."""
  groups = {}
  for fam_name, fam in eg.FAMILIES.items():
    if fam.seed is None:
      continue
    for name in gc.names(fam_name + '_'):
      g = gc.load(name)
      key = [fam_name]
      for k in fam.inputs:
        if k == 'actions' or (k == fam.seed[1] and k != 'config'):
          continue
        if k == 'config':           # everything but the seed it holds
          key.append(json.dumps({c: v for c, v in gc.config_of(g).items() if c != 'seed'},
                                sort_keys=True))
        else:
          key.append(bytes(np.ascontiguousarray(g[k])))
      groups.setdefault(tuple(key), []).append(name)
  return [(key[0], names) for key, names in groups.items()]


FAMILY_GROUPS = _family_goldens()


def _replay_group(game, goldens, seeds, rewards_f64):
  """Goldens[i] on env i of one engine of `game` beside DISTRACTORS envs: built with another
  rng_seed, reset(mask, seeds) on the golden envs, then each golden's actions through play(),
  every frame's board, reward, has_reward, discount and done compared."""
  n = len(goldens)
  B = n + DISTRACTORS
  eng = batched.BatchedEngine([game], batch=B, rng_seed=4242)
  eng.its_showtime()
  rs = np.random.RandomState(1)
  for _ in range(3):                   # the distractors are mid-episode
    eng.play(torch.from_numpy(rs.randint(0, 5, size=B).astype(np.int32)).cuda())
  mask = torch.zeros(B, dtype=torch.uint8, device='cuda')
  mask[:n] = 1
  all_seeds = list(seeds) + [123] * DISTRACTORS
  before = eng.board[n:].clone(), eng.rng[n:].clone()
  eng.reset(mask, seeds=all_seeds)
  assert torch.equal(eng.board[n:], before[0]) and torch.equal(eng.rng[n:], before[1])
  T = max(len(g['boards']) for g in goldens)
  got = {k: [] for k in ('boards', 'reward', 'has_reward', 'discount', 'done')}
  for t in range(T):
    got['boards'].append(eng.board[:n].cpu().numpy())
    got['reward'].append(eng.reward[:n].cpu().numpy())
    got['has_reward'].append(eng.has_reward[:n].cpu().numpy())
    got['discount'].append(eng.discount[:n].cpu().numpy())
    got['done'].append(eng.done[:n].cpu().numpy())
    if t == T - 1:
      break
    acts = rs.randint(0, 5, size=B).astype(np.int32)
    for e, g in enumerate(goldens):
      acts[e] = int(g['actions'][t]) if t < len(g['actions']) else 0
    eng.play(torch.from_numpy(acts).cuda())
  for e, g in enumerate(goldens):
    T_e = len(g['boards'])
    has = np.array([row[e] for row in got['has_reward'][:T_e]])
    assert np.array_equal(np.array([row[e] for row in got['boards'][:T_e]]), g['boards']), e
    assert np.array_equal(has, g['has_reward']), e
    want = g['reward_f64'] if rewards_f64 else g['reward']
    reward = np.array([row[e] for row in got['reward'][:T_e]])
    assert np.array_equal(reward[has == 1], want[has == 1]), e
    assert np.array_equal(np.array([row[e] for row in got['discount'][:T_e]], np.float64),
                          g['discount']), e
    assert np.array_equal(np.array([row[e] for row in got['done'][:T_e]]) != 0,
                          g['game_over'] != 0), e


@pytest.mark.parametrize('family,names', FAMILY_GROUPS, ids=['+'.join(n) for _, n in FAMILY_GROUPS])
def test_seeded_reset_replays_example_goldens(global_generators, family, names):  # noqa: F811
  fam = eg.FAMILIES[family]
  goldens = [gc.load(name) for name in names]
  make_env, _ = fam.facade(names[0], goldens[0])
  game = lowering.lower(make_env())
  assert game.needs_rng
  seeds = [eg._seed(g, fam.seed[1]) for g in goldens]
  _replay_group(game, goldens, seeds, game.float_reward)


def _registered_groups():
  out = []
  for m in rg.MODULES:
    mod = rg.load(m + '.py')
    groups = {}
    for row in mod.CASES:
      if row[4] is not None:
        groups.setdefault((row[1], row[2]), []).append(row[0])
    out += [(m + '.py', names) for names in groups.values()]
  return out


REGISTERED_GROUPS = _registered_groups()


@pytest.fixture(scope='module')
def games(request):
  yield from rg.registered(request.param)


@pytest.mark.parametrize('games,names', REGISTERED_GROUPS, indirect=['games'],
                         ids=['+'.join(n) for _, n in REGISTERED_GROUPS])
def test_seeded_reset_replays_registered_goldens(games, global_generators, names):  # noqa: F811
  game_name, level, _ = rg.case(games, names[0])
  game = lowering.lower(games.GAMES[game_name](level))
  if not game.needs_rng:
    pytest.skip('%s draws nothing on the device' % game_name)
  goldens = []
  for name in names:
    g = dict(gc.load(name))
    if game_name in games.RAISES:      # the frames before the step that raised
      at = int(g['raised_at'][0])
      g['actions'] = g['actions'][:at]
    goldens.append(g)
  seeds = [rg.case(games, name)[2] for name in names]
  _replay_group(game, goldens, seeds, game.float_reward)


# ---- same engine, two ways --------------------------------------------------------------

@pytest.mark.parametrize('name', PROGRAMS)
def test_built_with_a_equals_reseeded_to_a(global_generators, drawn, name):  # noqa: F811
  B, a = 16, 9001
  one = batched.BatchedEngine([_game(name, drawn)], batch=B, rng_seed=a)
  two = batched.BatchedEngine([_game(name, drawn)], batch=B, rng_seed=31337)
  one.its_showtime()
  two.its_showtime()
  two.play(torch.ones(B, dtype=torch.int32, device='cuda'))
  two.reset(seeds=a)
  rs = np.random.RandomState(2)
  for t in range(65):
    for k in ('board', 'reward', 'has_reward', 'discount', 'done', 'rng', 'sprites', 'drapes'):
      assert torch.equal(getattr(one, k), getattr(two, k)), (t, k)
    acts = torch.from_numpy(rs.randint(0, 5, size=B).astype(np.int32)).cuda()
    one.play(acts)
    two.play(acts)


# ---- the constructor --------------------------------------------------------------------

@pytest.mark.parametrize('name', PROGRAMS)
def test_constructor_words_are_the_host_loops(global_generators, drawn, name):  # noqa: F811
  game = _game(name, drawn)
  B = 4099
  eng = batched.BatchedEngine([game], batch=B, rng_seed=11)
  assert np.array_equal(_words(eng), _host_words(game, range(11, 11 + B)))
  shard = batched.BatchedEngine([game], batch=99, rng_seed=11, env_offset=1000)
  assert np.array_equal(_words(shard), _words(eng)[1000:1099])
  top = batched.BatchedEngine([game], batch=3, rng_seed=2 ** 32 - 3)
  assert np.array_equal(_words(top), _host_words(game, [2 ** 32 - 3, 2 ** 32 - 2, 2 ** 32 - 1]))


def test_constructor_keeps_host_words_outside_32_bits(drawn):
  from pycolab_b200.games import apprehend
  eng = batched.BatchedEngine([apprehend.make_game()], batch=3, rng_seed=-2)
  assert np.array_equal(_words(eng)[:, 0], np.stack([batched._mt_state('python', s)
                                                     for s in (-2, -1, 0)]))


# ---- capture ----------------------------------------------------------------------------

def _run(eng, mask, seeds, actions):
  eng.reset(mask, seeds=seeds)
  for t in range(actions.shape[0]):
    eng.play(actions[t])


def _state(eng):
  return [t.clone() for t in (eng.board, eng.reward, eng.done, eng.discount, eng.rng,
                              eng.sprites, eng.plot)]


@pytest.mark.parametrize('name', ['t_maze', 'marauders'])
def test_captured_seeded_reset_replays_new_seeds(global_generators, drawn, name):  # noqa: F811
  B, T = 64, 100
  game = _game(name, drawn)
  graphed = batched.BatchedEngine([game], batch=B, rng_seed=5)
  eager = batched.BatchedEngine([game], batch=B, rng_seed=5)
  rs = np.random.RandomState(3)
  actions = torch.from_numpy(rs.randint(0, 5, size=(T, B)).astype(np.int32)).cuda()
  mask = torch.from_numpy((rs.rand(B) < 0.5).astype(np.uint8)).cuda()
  seeds = torch.from_numpy(rs.randint(0, 2 ** 32, size=B, dtype=np.int64)).cuda()
  for eng in (graphed, eager):
    eng.its_showtime()
  side = torch.cuda.Stream()
  side.wait_stream(torch.cuda.current_stream())
  with torch.cuda.stream(side):           # warm up every launch the graph holds
    _run(graphed, mask, seeds, actions[:2])
  torch.cuda.current_stream().wait_stream(side)
  _run(eager, mask, seeds.clone(), actions[:2])
  graph = torch.cuda.CUDAGraph()
  with torch.cuda.graph(graph):
    _run(graphed, mask, seeds, actions)
  for k in range(3):
    seeds.copy_(torch.from_numpy(rs.randint(0, 2 ** 32, size=B, dtype=np.int64)))
    graph.replay()
    _run(eager, mask, seeds.clone(), actions)
    _sync()
    for a, b in zip(_state(graphed), _state(eager)):
      assert torch.equal(a, b), k


# ---- counters ---------------------------------------------------------------------------

def test_seeded_reset_restarts_the_time_limit_and_the_return(global_generators, drawn):  # noqa: F811
  B, L, before = 8, 6, 3
  eng = batched.BatchedEngine([_game('marauders', drawn)], batch=B, rng_seed=3, time_limit=L,
                              track_episodes=True)
  mask = torch.zeros(B, dtype=torch.uint8, device='cuda')
  mask[::2] = 1
  picked = mask.cpu().bool()
  rs = np.random.RandomState(4)       # actions 0-3: no env quits (4 is marauders' quit)
  eng.its_showtime()
  for _ in range(before):
    eng.play(torch.from_numpy(rs.randint(0, 4, size=B).astype(np.int32)).cuda())
  eng.reset(mask, seeds=1000)
  ret = (eng.reward.double() * eng.has_reward.double()).cpu()
  for k in range(L + 1):
    frames, done = eng.frames().cpu(), eng.done.cpu()
    # the seeded envs count from their reset, the others from its_showtime (and restart
    # the step after their limit)
    other = before + k if before + k <= L else before + k - L - 1
    assert frames[picked].eq(k).all() and frames[~picked].eq(other).all(), k
    assert torch.equal(eng.episode_return.cpu()[picked], ret[picked]), k
    ended = (done[picked] != 0).tolist()
    assert ended == [k == L] * len(ended), k
    if k == L:
      assert done[picked].eq(_lib.DONE_TIME_LIMIT).all()
      break
    eng.play(torch.from_numpy(rs.randint(0, 4, size=B).astype(np.int32)).cuda())
    ret = ret + (eng.reward.double() * eng.has_reward.double()).cpu()
