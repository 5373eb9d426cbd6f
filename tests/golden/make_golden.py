"""Generate the example-game, research-game and fixture goldens in this directory from the
REAL reference.

Run in the build container (where /root/reference exists):

    python tests/golden/make_golden.py [family ...]

With no argument it writes every golden of the families of tests/example_games.py and
the fixture_* goldens; with family names (FAMILIES keys: scrolly, classic, ...) only
those families' goldens.  Every .npz written here holds the inputs (level art as uint8
arrays, action stream, RNG seed, entity configuration as JSON) and the outputs the
unmodified reference produced for them (board per frame, reward, discount, game_over,
sprite registers, crops).  The GPU box has no /root/reference: the `-m gpu` parity tests
and the oracle tests compare against these files.
"""

import json
import os
import random
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

import box_world_cases as bwc
import example_games as eg
import lp_rnn_cases as lc
import refdriver
import trajectory as tj
from pycolab_b200 import levels


def save(name, **arrays):
  path = os.path.join(HERE, name + '.npz')
  np.savez_compressed(path, **arrays)
  print('%-32s %8.1f KiB' % (name, os.path.getsize(path) / 1024.0))


def record(name, **inputs):
  """Plays example golden `name` on the reference env its family builds from `inputs`
  (tests/example_games.py), then saves the inputs, the fields the family records and the
  trajectory, in the family's order.  Returns what it saved."""
  got = dict(eg.play('reference', name, inputs), **inputs)
  # a trajectory key the family's keys already place keeps its place
  arrays = {k: got[k] for k in eg.family_of(name).keys + tj.TRAJECTORY}
  save(name, **arrays)
  return arrays


def json_u8(obj):
  return np.frombuffer(json.dumps(obj).encode(), np.uint8)


# ------------------------------------------------------- example-game goldens --

def scrolly(name, maze, board, beneath, actions):
  record(name, maze_art=tj.art_to_u8(maze), board_art=tj.art_to_u8(board),
         beneath=np.array([ord(beneath)], dtype=np.uint8),
         actions=np.array(actions, dtype=np.int32))


def scrollies():
  # BASELINE.json configs[0]: stock scrolly_maze, 1000 random-action steps.
  for level, T in ((0, 1000), (1, 400), (2, 400)):
    maze, board, beneath = refdriver.ref_stock_scrolly_art(level)
    rs = np.random.RandomState(100 + level)
    scrolly('scrolly_stock_L%d' % level, maze, board, beneath,
            rs.randint(0, 5, size=T).tolist())
  maze, board, beneath = refdriver.ref_stock_scrolly_art(0)
  scrolly('scrolly_stock_L0_quit', maze, board, beneath,
          np.random.RandomState(7).randint(0, 6, size=300).tolist())
  for seed in (0, 1):
    maze, board, beneath = levels.scrolly_maze_level(seed)
    acts = np.random.RandomState(seed).choice(
        [0, 1, 2, 3, 4], size=300, p=[.3, .15, .3, .15, .1]).tolist()
    scrolly('scrolly_gen64_s%d' % seed, maze, board, beneath, acts)
  # Board shapes the step kernels branch on (tests/scrolly_shapes.py): 11x33 (3 segments
  # per row), 33x63 (a ragged second round of rows, partial high half) and 65x64 (a
  # third round).
  import scrolly_shapes as ss
  for name in ('11x33', '33x63', '65x64'):
    maze, board, beneath = ss.shape_level(name, 0)
    actions = np.random.RandomState(len(name)).choice([0, 1, 2, 3, 4], size=300,
                                                      p=[.2, .2, .27, .27, .06])
    scrolly('scrolly_shape%s' % name, maze, board, beneath, actions.tolist())


def warehouse(name, art, wlb, actions):
  chars = [c for c in '1234567890' if c in ''.join(art)] + ['P']
  wlb_arr = (np.array([[ord(wlb)]], dtype=np.uint8) if isinstance(wlb, str)
             else tj.art_to_u8(wlb))
  record(name, art=tj.art_to_u8(art), what_lies_beneath=wlb_arr,
         sprite_chars=np.frombuffer(''.join(chars).encode(), dtype=np.uint8),
         actions=np.array(actions, dtype=np.int32))


def warehouses():
  for level in (0, 1, 2):
    art, wlb = refdriver.ref_stock_warehouse_art(level)
    warehouse('warehouse_stock_L%d' % level, art, wlb,
              np.random.RandomState(200 + level).randint(0, 5, size=600).tolist())
  art = levels.warehouse_level(3)
  warehouse('warehouse_gen80_s3', art, ' ',
            np.random.RandomState(3).randint(0, 4, size=250).tolist())


def marauder(name, seed, actions, art=None):
  art = refdriver.ref_stock_marauders_art() if art is None else art
  record(name, art=tj.art_to_u8(art), rng_seed=np.array([seed], dtype=np.int64),
         actions=np.array(actions, dtype=np.int32))


def marauders():
  for seed in (0, 1, 2):
    marauder('marauders_stock_s%d' % seed, seed,
              np.random.RandomState(300 + seed).randint(0, 4, size=1000).tolist())
  # the largest board the step kernel takes
  marauder('marauders_shape32x64', 5, np.random.RandomState(5).randint(0, 4, size=400).tolist(),
            art=levels.marauders_level(32, 64))


def better_scrolly(name, level, T=400):
  """better_scrolly_maze stock level + its three croppers (player view with an
  initial offset and no padding, patroller view padded with (None, 3) margins,
  fixed teaser window)."""
  art, offset, teaser = refdriver.ref_better_scrolly_stock(level)
  rs = np.random.RandomState(700 + level)
  actions = rs.randint(0, 5, size=T).tolist()
  record(name, art=tj.art_to_u8(art), starter_offset=np.array(offset, dtype=np.int32),
         teaser_corner=np.array(teaser, dtype=np.int32),
         actions=np.array(actions, dtype=np.int32))


def better_scrollies():
  for level in (0, 1, 2):
    better_scrolly('better_stock_L%d' % level, level)


def cropper(name, pad, margins, offset, saccade, T=300):
  maze, board, beneath = levels.scrolly_maze_level(5, world_shape=(65, 65),
                                                   board_shape=(32, 32))
  rs = np.random.RandomState(11)
  actions = rs.randint(0, 5, size=T)
  cfg = dict(rows=9, cols=9, pad=pad, margins=list(margins),
             offset=None if offset is None else list(offset), saccade=saccade)
  record(name, maze_art=tj.art_to_u8(maze), board_art=tj.art_to_u8(board),
         beneath=np.array([ord(beneath)], dtype=np.uint8),
         config=json_u8(cfg), actions=actions.astype(np.int32))


def croppers():
  cropper('crop_ego_pad', ' ', (None, None), None, True)
  cropper('crop_margins_nopad', None, (2, 3), None, True)
  cropper('crop_margins_pad_offset', ' ', (2, 3), (1, -2), False)


def classics():
  """examples/classics games; rewards are Python floats there, so the goldens also
  record the reward's type."""
  for kind in ('four_rooms', 'cliff_walk', 'chain_walk'):
    n_actions = 3 if kind == 'chain_walk' else 6
    for which, art in (('stock', None), ('other', levels.classic_level(kind))):
      actions = np.random.RandomState(len(kind) + len(which)).randint(0, n_actions, size=1200)
      record('classic_%s_%s' % (kind, which),
             art=tj.art_to_u8(art or refdriver.ref_classic_art(kind)),
             kind=np.frombuffer(kind.encode(), dtype=np.uint8),
             actions=actions.astype(np.int32))


def fluvials():
  """examples/fluvial_natation.py; also records the (mutable) backdrop curtain."""
  for which, art in (('stock', refdriver.ref_fluvial_art()), ('other', levels.fluvial_level())):
    actions = np.random.RandomState(len(which)).choice([0, 1, 2], size=800, p=[.2, .6, .2])
    record('fluvial_%s' % which, art=tj.art_to_u8(art), actions=actions.astype(np.int32))


# Level 0 played to the cranachan: two aperture pairs, two teleports, reward 1.
APERTURE_SCRIPT_L0 = [8, 7, 1, 1, 2, 1, 1, 1, 1, 1, 6, 8, 3, 3, 1, 1, 1, 3, 4, 0]


def apertures():
  """examples/aperture.py stock levels; records the player registers and the aperture
  curtain each frame."""
  for level in (0, 1, 2):
    rs = np.random.RandomState(40 + level)
    actions = rs.choice(list(range(10)), size=900,
                        p=[.14, .14, .14, .14, .04, .1, .1, .1, .095, .005])
    record('aperture_stock_L%d' % level, art=tj.art_to_u8(refdriver.ref_aperture_art(level)),
           actions=actions.astype(np.int32))
  record('aperture_script_L0', art=tj.art_to_u8(refdriver.ref_aperture_art(0)),
         actions=np.array(APERTURE_SCRIPT_L0, dtype=np.int32))


def hellos():
  """examples/hello_world.py: stock art, random actions 0-5 (4 quits, 5 is a no-op)."""
  refdriver._import()
  from pycolab.examples import hello_world as ref_hello
  for seed in range(2):
    rs = np.random.RandomState(600 + seed)
    actions = rs.choice([0, 1, 2, 3, 4, 5], size=400, p=[.22, .22, .22, .22, .02, .10])
    record('hello_stock_s%d' % seed, art=tj.art_to_u8(ref_hello.HELLO_ART),
           actions=actions.astype(np.int32))


def apprehends():
  """examples/apprehend.py: stock art; `random.seed` fixes the global stream the ball
  sprites draw their slopes from (one draw per episode), actions 0-2 (2 = stay put)."""
  refdriver._import()
  from pycolab.examples import apprehend as ref_app
  for seed in range(3):
    rs = np.random.RandomState(700 + seed)
    actions = rs.randint(0, 3, size=300)
    traj = record('apprehend_stock_s%d' % seed, art=tj.art_to_u8(ref_app.GAME_ART),
                  actions=actions.astype(np.int32), random_seed=np.array([700 + seed]))
    print('  apprehend_stock_s%d: %d episodes, reward sum %d' % (
        seed, int(traj['game_over'].sum()), int(traj['reward'].sum())))


def shockwave(cases, first_seed=0):
  """examples/shockwave.py levels; `np.random.seed` fixes the global stream the impact
  points come from; actions 0-4 (4 = none of the keys), biased upwards so that some
  episodes are won."""
  for seed, (tag, art) in enumerate(cases, first_seed):
    name = 'shockwave_%s' % tag
    g = dict(art=tj.art_to_u8(art), numpy_seed=np.array([800 + seed]))
    make = eg.family_of(name).reference(name, g)[0]
    # pass 1: a climbing policy that looks at the reference env (up when the cell
    # above is free, else sideways; sometimes waits) chooses the actions ...
    rs = np.random.RandomState(800 + seed)
    np.random.seed(800 + seed)
    actions, env = [], make()
    env.its_showtime()
    for _ in range(500):
      if env.game_over:
        env = make()
        env.its_showtime()
        actions.append(int(rs.randint(0, 5)))        # ignored by the protocol
        continue
      r, c = env.things['P'].position
      up_free = r > 0 and art[r - 1][c] != '='
      a = int(rs.choice([0, 1, 2, 3, 4], p=[.7, .08, .08, .1, .04] if up_free
                        else [.05, .4, .4, .1, .05]))
      actions.append(a)
      env.play(a)
    # ... pass 2 replays them through the shared trajectory protocol
    traj = record(name, actions=np.array(actions, dtype=np.int32), **g)
    print('  %s: %d episodes, wins %d, deaths %d' % (
        name, int(traj['game_over'].sum()), int((traj['reward'] == 1).sum()),
        int((traj['reward'] == -1).sum())))


def shockwaves():
  """The stock level, two generated ones (12x15, 20x40) and the largest board the step
  kernel takes, 32x64."""
  refdriver._import()
  from pycolab.examples import shockwave as ref_shock
  shockwave([('stock', ref_shock.LEVELS[0]),
              ('g12x15', levels.shockwave_level(1, safety_density=0.5)),
              ('g20x40', levels.shockwave_level(2, 20, 40, 0.6))])
  shockwave([('g32x64', levels.shockwave_level(96, 32, 64, 0.5))], first_seed=3)


def ordeals():
  """examples/ordeal.py through the reference's own Story (cropped observations,
  summed rewards across chapter crossings, discounts, chapter names, has_sword)."""
  import ordeal_cases
  for name, actions in sorted(ordeal_cases.scripts().items()):
    traj = record(name, actions=np.array(actions, dtype=np.int32))
    print('  %s: %d steps, chapters %s, reward sum %s' % (
        name, len(traj['boards']) - 1, sorted(set(traj['chapters'].tolist())),
        traj['reward'].sum()))


def stories():
  """Reference Stories of classics chapters (example_games._story), each played to its
  end (then rebuilt, like any env of the trajectory protocol)."""
  rs = np.random.RandomState(77)
  a1 = rs.randint(0, 5, size=700)
  a1[rs.random_sample(700) < 0.01] = 5              # quit now and then: next chapter
  a2 = rs.randint(0, 4, size=900)
  record('story_classics_list', actions=(a1 % 4).astype(np.int32))
  record('story_classics_cropped', actions=a2.astype(np.int32))


# ----------------------------------------------------------- research goldens --

def t_mazes():
  """research/lp-rnn/t_maze.py on its own art: `random.seed` and `np.random.seed` fix the
  streams the cue side and the speckle are drawn from at every make_game."""
  ref = lc.ref_module('t_maze')
  for name, level, cue_after, timeout, delay, limbo, seed, T in lc.T_MAZE_CASES:
    actions = lc.t_maze_policy(900 + seed, limbo, T)
    if name.endswith('_quit'):
      actions = [6 if a == 5 and i % 3 == 0 else a for i, a in enumerate(actions)]
    config = dict(level=level, cue_after_teleport=cue_after, timeout_frames=timeout,
                  teleport_delay=delay, limbo_time=limbo, seed=900 + seed)
    traj = record(name, maze_art=tj.art_to_u8(ref.MAZE_ART), cue_art=tj.art_to_u8(ref.CUE_ART),
                  actions=np.array(actions, dtype=np.int32), config=json_u8(config))
    r = traj['reward_f64']
    print('  %s: %d episodes, +1 %d, -1 %d, quits/timeouts %d' % (
        name, int(traj['game_over'].sum()), int((r > 0.5).sum()), int((r < -0.5).sum()),
        int(traj['game_over'].sum()) - int((np.abs(r) > 0.5).sum())))


def lp_rnn(name, art, args, seed, T, policy):
  """A Cued Catch or Sequence Recall golden: `random.seed` fixes the stream the game draws
  from.  Pass 1 lets policy(env) choose T actions on the reference env, pass 2 records them."""
  g = dict(art=tj.art_to_u8(art), config=json_u8(dict(args=list(args), seed=900 + seed)))
  random.seed(900 + seed)
  actions = lc.closed_loop(eg.family_of(name).reference(name, g)[0], policy, T)
  return record(name, actions=np.array(actions, dtype=np.int32), **g)


def cued_catches():
  """research/lp-rnn/cued_catch.py, shimmed (tests/lp_rnn_cases.py)."""
  ref = lc.ref_module('cued_catch')
  for name, art, args, seed, T, kw in lc.CUED_CATCH_CASES:
    art = list(ref.GAME_ART) if art is None else lc.small_cued_catch_art()
    traj = lp_rnn(name, art, args, seed, T,
                  lc.cued_catch_policy(np.random.RandomState(seed), **kw))
    print('  %s: %d episodes, reward sum %.3f, float frames %d' % (
        name, int(traj['game_over'].sum()), float(np.nansum(traj['reward_f64'])),
        int((traj['reward_type'] == 2).sum())))


def sequence_recalls():
  """research/lp-rnn/sequence_recall.py, shimmed (tests/lp_rnn_cases.py)."""
  ref = lc.ref_module('sequence_recall')
  for name, art, args, seed, T, kw in lc.SEQUENCE_RECALL_CASES:
    art = list(ref.GAME_ART) if art == 'ref' else levels.sequence_recall_art(*art)
    centre = tuple(int(x[0]) for x in np.where(tj.art_to_u8(art) == ord('P')))
    traj = lp_rnn(name, art, args, seed, T,
                  lc.sequence_recall_policy(np.random.RandomState(seed), centre, **kw))
    r = traj['reward_f64']
    print('  %s: %d episodes, +1 %d, wrong %d' % (
        name, int(traj['game_over'].sum()), int((r > 0.9).sum()), int((r == -0.005).sum())))


def box_worlds():
  """research/box_world: the level the reference generates from RandomState(seed) at every
  (re)start.  Pass 1 lets the scripted player of tests/box_world_cases.py choose the actions
  on the reference env, pass 2 records them."""
  for name, seed, grid_size, max_steps, modes, T in bwc.CASES:
    g = dict(config=json_u8(dict(seed=seed, grid_size=grid_size, max_num_steps=max_steps,
                                 modes=list(modes))))
    make = eg.family_of(name).reference(name, g)[0]
    first = make()
    art = [bytes(r).decode() for r in first.its_showtime()[0].board]
    distractors = list(first.things['.'].distractors)
    traj = record(name, art=tj.art_to_u8(art),
                  distractors=np.array(distractors, np.int32).reshape(-1, 2),
                  actions=np.array(bwc.drive(make, distractors, modes, T, seed), np.int32), **g)
    r = traj['reward_f64']
    print('  %s: %d episodes, rewards %s' % (
        name, int(traj['game_over'].sum()), sorted(set(float(v) for v in r[~np.isnan(r)]))))


# The makers of each family of tests/example_games.py.
MAKERS = dict(scrolly=scrollies, warehouse=warehouses, marauders=marauders,
              better=better_scrollies, crop=croppers, classic=classics, fluvial=fluvials,
              aperture=apertures, hello=hellos, apprehend=apprehends, shockwave=shockwaves,
              ordeal=ordeals, story=stories, t_maze=t_mazes, cued_catch=cued_catches,
              sequence_recall=sequence_recalls, box_world=box_worlds)


# ------------------------------------------------------------ fixture goldens --

def fixture_walkers(name, seed, T=300):
  rs = np.random.RandomState(seed)
  H, W = int(rs.randint(5, 12)), int(rs.randint(5, 14))
  art = np.full((H, W), ord(' '), dtype=np.uint8)
  art[rs.random_sample((H, W)) < 0.25] = ord('#')
  art[rs.random_sample((H, W)) < 0.1] = ord('%')
  free = np.argwhere(art == ord(' '))
  picks = free[rs.permutation(len(free))[:3]]
  for ch, (r, c) in zip('abc', picks):
    art[r, c] = ord(ch)
  walkers = {
      'a': dict(impassable='#', confined=bool(rs.randint(2))),
      'b': dict(impassable='#%a', confined=bool(rs.randint(2))),
      'c': dict(impassable='', confined=False),
  }
  schedule = [['a'], ['b', 'c']] if rs.randint(2) else [['a', 'b', 'c']]
  z_order = ''.join(rs.permutation(list('abc')))
  art_l = tj.u8_to_art(art)
  motions = rs.randint(0, 9, size=(T, 3)).astype(np.int32)
  sprites = []
  traj = tj.run_trajectory(
      lambda: refdriver.ref_fixture(art_l, ' ', walkers,
                                    update_schedule=schedule, z_order=z_order),
      motions,
      convert_action=lambda m: refdriver.fixture_actions_to_ref(
          {ch: int(v) for ch, v in zip('abc', m)}),
      on_frame=lambda env, out: sprites.append(tj.sprite_rows(env, 'abc')))
  cfg = dict(walkers=walkers, scrollys={}, drapes='', schedule=schedule,
             z_order=z_order, what_lies_beneath=' ', action_chars='abc')
  save(name, art=art, config=json_u8(cfg),
       actions=motions, sprites=np.array(sprites, dtype=np.int32), **traj)


def fixture_scrolly(name, seed, margins, second_ego, T=400):
  rs = np.random.RandomState(1000 + seed)
  PH, PW, H, W = 17, 23, 8, 11
  pattern = rs.random_sample((PH, PW)) < 0.2
  pattern2 = rs.random_sample((PH, PW)) < 0.1
  corner = (int(rs.randint(0, PH - H + 1)), int(rs.randint(0, PW - W + 1)))
  art = np.full((H, W), ord(' '), dtype=np.uint8)
  art[3, 4] = ord('P')
  art[5, 7] = ord('q')
  art_l = tj.u8_to_art(art)
  walkers = {'P': dict(impassable='#', egocentric=True),
             'q': dict(impassable='#', egocentric=bool(second_ego))}
  scrollys = {'#': dict(pattern=pattern, corner=corner, margins=margins),
              '@': dict(pattern=pattern2, corner=corner, margins=margins)}
  schedule = [['#'], ['P', 'q'], ['@']]
  motions = rs.randint(0, 9, size=(T,)).astype(np.int32)
  sprites, curtains = [], []

  def on_frame(env, out):
    sprites.append(tj.sprite_rows(env, 'Pq'))
    curtains.append(np.stack([env.things['#'].curtain.copy(),
                              env.things['@'].curtain.copy()]))

  env = refdriver.ref_fixture(art_l, ' ', walkers, scrollys,
                              update_schedule=schedule, z_order='@#Pq')
  out = env.its_showtime()
  boards = [tj.board_of(out[0]).copy()]
  on_frame(env, out)
  used = []
  for m in motions:
    try:
      out = env.play(refdriver.fixture_actions_to_ref(int(m)))
    except RuntimeError:
      break                         # reference rejects a (0,0)-clipped order
    used.append(int(m))
    boards.append(tj.board_of(out[0]).copy())
    on_frame(env, out)
  cfg = dict(
      walkers=walkers,
      scrollys={ch: dict(corner=list(corner),
                         margins=None if margins is None else list(margins))
                for ch in '#@'},
      drapes='', schedule=schedule, z_order='@#Pq', what_lies_beneath=' ',
      action_chars='')
  save(name, art=art, config=json_u8(cfg),
       pattern_hash=pattern.astype(np.uint8), pattern_at=pattern2.astype(np.uint8),
       actions=np.array(used, dtype=np.int32), boards=np.stack(boards),
       sprites=np.array(sprites, dtype=np.int32),
       curtains=np.stack(curtains).astype(np.uint8))


def fixture_groups(name, seed, margins, T=400):
  """Two scrolling groups at once (protocols/scrolling.py:198-241): group 'one' =
  Scrolly '#' + egocentric walker P, group 'two' = Scrolly '@' + egocentric walker q;
  every step each group gets its own random motion, so the two windows scroll
  independently and each walker obeys only its own group's orders."""
  rs = np.random.RandomState(2000 + seed)
  PH, PW, H, W = 17, 23, 8, 11
  pattern = rs.random_sample((PH, PW)) < 0.2
  pattern2 = rs.random_sample((PH, PW)) < 0.1
  corner = (int(rs.randint(0, PH - H + 1)), int(rs.randint(0, PW - W + 1)))
  corner2 = (int(rs.randint(0, PH - H + 1)), int(rs.randint(0, PW - W + 1)))
  art = np.full((H, W), ord(' '), dtype=np.uint8)
  art[3, 4] = ord('P')
  art[5, 7] = ord('q')
  art_l = tj.u8_to_art(art)
  walkers = {'P': dict(impassable='#', egocentric=True, group='one'),
             'q': dict(impassable='@', egocentric=True, group='two')}
  scrollys = {'#': dict(pattern=pattern, corner=corner, margins=margins, group='one'),
              '@': dict(pattern=pattern2, corner=corner2, margins=margins, group='two')}
  schedule = [['#', '@'], ['P', 'q']]
  motions = rs.randint(0, 9, size=(T, 2)).astype(np.int32)      # (group one, group two)
  sprites, curtains = [], []

  def on_frame(env, out):
    sprites.append(tj.sprite_rows(env, 'Pq'))
    curtains.append(np.stack([env.things['#'].curtain.copy(),
                              env.things['@'].curtain.copy()]))

  env = refdriver.ref_fixture(art_l, ' ', walkers, scrollys,
                              update_schedule=schedule, z_order='@#Pq')
  out = env.its_showtime()
  boards = [tj.board_of(out[0]).copy()]
  on_frame(env, out)
  used = []
  for m1, m2 in motions:
    act = {'#': int(m1), 'P': int(m1), '@': int(m2), 'q': int(m2)}
    try:
      out = env.play(refdriver.fixture_actions_to_ref(act))
    except RuntimeError:
      break                         # reference rejects a (0,0)-clipped order
    used.append([int(m1), int(m2)])
    boards.append(tj.board_of(out[0]).copy())
    on_frame(env, out)
  cfg = dict(
      walkers=walkers,
      scrollys={'#': dict(corner=list(corner), group='one',
                          margins=None if margins is None else list(margins)),
                '@': dict(corner=list(corner2), group='two',
                          margins=None if margins is None else list(margins))},
      drapes='', schedule=schedule, z_order='@#Pq', what_lies_beneath=' ',
      action_chars='', motion_of=dict([('#', 0), ('P', 0), ('@', 1), ('q', 1)]))
  save(name, art=art, config=json_u8(cfg),
       pattern_hash=pattern.astype(np.uint8), pattern_at=pattern2.astype(np.uint8),
       actions=np.array(used, dtype=np.int32).reshape(-1, 2), boards=np.stack(boards),
       sprites=np.array(sprites, dtype=np.int32),
       curtains=np.stack(curtains).astype(np.uint8))
  print('  %s: %d steps' % (name, len(used)))


def fixture_unoccluded(name, seed, T=120):
  """occlusion_in_layers=False (BaseUnoccludedObservationRenderer,
  rendering.py:187-301): per-frame layers of every character."""
  rs = np.random.RandomState(6000 + seed)
  PH, PW, H, W = 13, 17, 7, 10
  pattern = rs.random_sample((PH, PW)) < 0.25
  corner = (int(rs.randint(0, PH - H + 1)), int(rs.randint(0, PW - W + 1)))
  art = np.full((H, W), ord(' '), dtype=np.uint8)
  art[rs.random_sample((H, W)) < 0.15] = ord('.')
  art[1:4, 2:7] = ord('%')
  art[3, 4] = ord('P')
  art[5, 7] = ord('q')
  art_l = tj.u8_to_art(art)
  walkers = {'P': dict(impassable='#', egocentric=True),
             'q': dict(impassable='', confined=True)}
  scrollys = {'#': dict(pattern=pattern, corner=corner, margins=(2, 3))}
  schedule = [['#'], ['P', 'q', '%']]
  z_order = 'q%#P'
  env = refdriver.ref_fixture(art_l, ' ', walkers, scrollys, drapes='%',
                              update_schedule=schedule, z_order=z_order,
                              occlusion_in_layers=False)
  out = env.its_showtime()
  chars = ''.join(sorted(out[0].layers))
  boards, layers = [], []

  def record(out):
    boards.append(tj.board_of(out[0]).copy())
    layers.append(np.stack([np.array(out[0].layers[c], dtype=bool) for c in chars]))
  record(out)
  motions = rs.randint(0, 9, size=T)
  for m in motions:
    record(env.play(refdriver.fixture_actions_to_ref(int(m))))
  cfg = dict(walkers=walkers,
             scrollys={'#': dict(corner=list(corner), margins=[2, 3])},
             drapes='%', schedule=schedule, z_order=z_order, what_lies_beneath=' ',
             action_chars='', layer_chars=chars)
  save(name, art=art, config=json_u8(cfg),
       pattern_hash=pattern.astype(np.uint8), actions=motions.astype(np.int32),
       boards=np.stack(boards), layers=np.stack(layers).astype(np.uint8))


def fixture_directives(name, seed, T=250):
  """Walkers + a static drape with Plot directives injected through
  test_things.post_update: rewards, z-order changes, a final termination."""
  tt = refdriver._import()['test_things']
  rs = np.random.RandomState(5000 + seed)
  H, W = 7, 9
  art = np.full((H, W), ord(' '), dtype=np.uint8)
  art[rs.random_sample((H, W)) < 0.2] = ord('#')
  art[2:5, 3:6] = ord('%')                      # static drape region
  for ch, (r, c) in zip('abc', [(1, 1), (5, 7), (3, 4)]):
    art[r, c] = ord(ch)
  art_l = tj.u8_to_art(art)
  walkers = {'a': dict(impassable='#', confined=True),
             'b': dict(impassable='#c', confined=False),
             'c': dict(impassable='', confined=True)}
  schedule = [['a', '%'], ['b', 'c']]
  order = 'a%bc'
  z_order = ''.join(rs.permutation(list(order)))
  engine = refdriver.ref_fixture(art_l, ' ', walkers, drapes='%',
                                 update_schedule=schedule, z_order=z_order)
  out = engine.its_showtime()
  boards = [tj.board_of(out[0]).copy()]
  reward, has_reward, discount, over = [0], [0], [float(out[2])], [0]
  rows, z_orders = [], [list(map(ord, engine.z_order))]
  for t in range(T):
    motions = {ch: int(rs.randint(0, 9)) for ch in 'abc'}
    r = int(rs.randint(-5, 50)) if rs.random_sample() < 0.3 else None
    z = None
    if rs.random_sample() < 0.25:
      this = order[int(rs.randint(4))]
      that = None if rs.random_sample() < 0.3 else order[int(rs.randint(4))]
      if that != this:
        z = (this, that)
    term = (t == T - 1)

    def inject(actions, board, layers, backdrop, things, the_plot, r=r, z=z, term=term):
      if r is not None:
        the_plot.add_reward(r)
      if term:
        the_plot.terminate_episode()
      if z is not None:
        the_plot.change_z_order(*z)
    tt.post_update(engine, 'c', inject)
    out = engine.play(refdriver.fixture_actions_to_ref(motions))
    row = [motions.get(ch, 8) for ch in order]
    row += [-(2 ** 31) if r is None else r, int(term)]
    row += [-1, 0] if z is None else [ord(z[0]), 0 if z[1] is None else ord(z[1])]
    rows.append(row)
    boards.append(tj.board_of(out[0]).copy())
    reward.append(0 if out[1] is None else int(out[1]))
    has_reward.append(0 if out[1] is None else 1)
    discount.append(float(out[2]))
    over.append(int(engine.game_over))
    z_orders.append(list(map(ord, engine.z_order)))
  cfg = dict(walkers=walkers, scrollys={}, drapes='%', schedule=schedule,
             z_order=z_order, what_lies_beneath=' ', action_chars=order)
  save(name, art=art, config=json_u8(cfg),
       actions=np.array(rows, dtype=np.int64), boards=np.stack(boards),
       reward=np.array(reward, dtype=np.int64),
       has_reward=np.array(has_reward, dtype=np.uint8),
       discount=np.array(discount, dtype=np.float64),
       game_over=np.array(over, dtype=np.uint8),
       z_orders=np.array(z_orders, dtype=np.uint8))


def fixtures():
  for seed in range(6):
    fixture_walkers('fixture_walkers_%d' % seed, seed)
  for seed, margins, ego2 in ((0, (2, 3), 0), (1, None, 1), (2, (1, 1), 0),
                              (3, None, 0), (4, (2, 2), 1), (5, (1, 2), 1)):
    fixture_scrolly('fixture_scrolly_%d' % seed, seed, margins, ego2)
  for seed in range(3):
    fixture_directives('fixture_directives_%d' % seed, seed)
  for seed in range(2):
    fixture_unoccluded('fixture_unoccluded_%d' % seed, seed)
  for seed, margins in ((0, (2, 3)), (1, None), (2, (1, 2))):
    fixture_groups('fixture_groups_%d' % seed, seed, margins)


def main():
  assert refdriver.available(), '/root/reference is required'
  families = sys.argv[1:]
  unknown = sorted(set(families) - set(MAKERS))
  assert not unknown, 'no family %s: the families are %s' % (unknown, sorted(MAKERS))
  for family in families or MAKERS:
    MAKERS[family]()
  if not families:
    fixtures()


if __name__ == '__main__':
  main()
