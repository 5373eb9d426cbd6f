"""Shared pieces of the lp-rnn tests and golden fixtures (t_maze, Cued Catch, Sequence
Recall): the reference's own modules (loaded by path), the two shims that let Cued Catch and
Sequence Recall run on Python 3 with NumPy 2 without touching their source, the golden cases
and their policies, and the per-frame state the goldens record.

The shims:
  * Cued Catch compares None with ints the Python 2 way (None below everything):
    `the_plot.get('last_ball_reset') > last_reset` and `0 <= cue` in `_show_cue(None)`.
    Seeding the_plot['last_ball_reset'] = -inf and mapping `_show_cue(None)` to
    `_show_cue(-1)` reproduce it.
  * Sequence Recall subtracts boolean arrays (`curtain[:] -= mask`), which NumPy 1 did as
    XOR.  Viewing the mask drape's curtain as an ndarray whose `__isub__` is `^=` reproduces
    it.
"""

import importlib.util
import os

import numpy as np

import refdriver

NEVER = -(2 ** 31)
NO_TIMEOUT = 0x7fffffff


def ref_module(name):
  """research/lp-rnn/<name>.py of the reference, loaded by path (not a package)."""
  refdriver._import()
  path = os.path.join(refdriver.REFERENCE_ROOT, 'pycolab', 'examples', 'research', 'lp-rnn',
                      name + '.py')
  spec = importlib.util.spec_from_file_location('ref_%s_lp_rnn' % name, path)
  module = importlib.util.module_from_spec(spec)
  spec.loader.exec_module(module)
  return module


class XorSubArray(np.ndarray):
  """NumPy 1's boolean `a -= b`: XOR."""

  def __isub__(self, other):
    np.bitwise_xor(self, other, out=self)
    return self


def shim_cued_catch(engine):
  engine.the_plot['last_ball_reset'] = -float('inf')
  cue = engine.things['Q']
  show = cue._show_cue
  cue._show_cue = lambda c=None: show(-1 if c is None else c)
  return engine


def shim_sequence_recall(engine):
  mask = engine.things['M']
  mask._c_u_r_t_a_i_n = mask._c_u_r_t_a_i_n.view(XorSubArray)
  return engine


def with_art(module, art, make):
  """make() with the module's GAME_ART replaced by `art` for the call (make_game reads it)."""
  saved = module.GAME_ART
  module.GAME_ART = list(art)
  try:
    return make()
  finally:
    module.GAME_ART = saved


# -------------------------------------------------------------------------------- t_maze --

# (name, level, cue_after_teleport, timeout_frames, teleport_delay, limbo_time, seed, T)
T_MAZE_CASES = (
    ('t_maze_L0_limbo4', 0, False, -1, 0, 4, 0, 700),
    ('t_maze_L1_delay5_cue', 1, True, -1, 5, 0, 1, 700),
    ('t_maze_L2_limbo10_timeout', 2, False, 90, 5, 10, 2, 700),
    ('t_maze_L3_cue_limbo2', 3, True, -1, 0, 2, 3, 700),
    ('t_maze_L4_delay5_limbo4', 4, False, 300, 5, 4, 4, 900),
    ('t_maze_L5_quit', 5, True, -1, 0, 10, 5, 900),
)


def t_maze_policy(seed, limbo_time, T):
  """Actions that reach the goals: north onto the teleporter, wait out limbo, then along the
  hallway to one side (drawn per episode) and down the corridor; some noise, some quits."""
  rs = np.random.RandomState(seed)
  out = []
  while len(out) < T:
    side = int(rs.choice([3, 4]))
    episode = [1, 1, 1] + [5] * (max(limbo_time, 0) + 3) + [side] * 100 + [2] * 8
    episode = [int(rs.randint(1, 6)) if rs.random_sample() < 0.05 else a for a in episode]
    out += episode
  return out[:T]


# ---------------------------------------------------------------------------- Cued Catch --

# (name, art (None = the reference's), make_game args, seed, T, policy kwargs)
CUED_CATCH_CASES = (
    ('cued_catch_paper', None, (10, 10, 100, False, 0.0, 40), 0, 1500, {}),
    ('cued_catch_free_trials', None, (3, 2, 12, False, 0.0, 3), 1, 400, {}),
    ('cued_catch_sigma', None, (2, 3, 10, False, 0.5, 2), 2, 500, {}),
    ('cued_catch_always', None, (2, 2, 8, True, 0.0, 0), 3, 300, {}),
    ('cued_catch_quit0', None, (2, 3, 20, False, 0.0, 0), 4, 300, dict(quit_every=67, quit_action=0)),
    ('cued_catch_quit4', None, (1, 1, 20, False, 1.5, 1), 5, 300, dict(quit_every=53, quit_action=4)),
    ('cued_catch_small_board', 'small', (3, 2, 15, True, 0.25, 1), 6, 500, {}),
)


def small_cued_catch_art():
  """5 x 14: a width that is no multiple of 4, 'Q' cells in row 0, balls in other columns,
  and fewer than 7 rows, so the bands 3:5 and -2: overlap."""
  from pycolab_b200 import levels
  return levels.cued_catch_art(5, 14, player=(1, 2), balls=((1, 9), (2, 12)),
                               cue_cells=((0, 0), (0, 5), (0, 13), (2, 7)))


def cued_catch_policy(rs, quit_every=0, quit_action=4):
  """Mostly moves to the correct ball's row (read from the env), sometimes the other way or
  nothing; every `quit_every`-th step quits."""
  count = [0]

  def act(env):
    count[0] += 1
    if quit_every and count[0] % quit_every == 0:
      return quit_action
    if rs.random_sample() < 0.25:
      return int(rs.choice([1, 2, 3, 5]))
    things = env.things
    which = env.the_plot.get('which_ball')
    ball = things['a' if which == 'top' else 'b']
    row = things['P'].position[0]
    return 1 if ball.position[0] < row else 2 if ball.position[0] > row else 3
  return act


def cued_catch_state(env):
  """[phase, first tick, choice, second tick, last reset, trials left, pairings bits,
  trials till reward, programming_complete, which_ball (0 unset, 1 top, 2 bottom),
  last_ball_reset (NEVER unset)] of a reference or facade Engine."""
  q, p, plot = env.things['Q'], env.things['P'], env.the_plot
  last = q._second_phase_last_reset
  lbr = plot.get('last_ball_reset')
  return [0 if q._phase == 'first' else 1, q._first_phase_tick, q._second_phase_cue_choice,
          q._second_phase_tick, NEVER if last == -float('inf') else last, q._num_trials_left,
          sum(1 << k for k, b in enumerate(q._cues_to_balls) if b == 'top'),
          p._trials_till_reward, 1 if plot.get('programming_complete') else 0,
          {None: 0, 'top': 1, 'bottom': 2}[plot.get('which_ball')],
          NEVER if lbr is None or lbr == -float('inf') else lbr]


def oracle_cued_catch_state(world):
  q, p, store = world.things['Q'].aux, world.things['P'].aux, world.plot.store
  lbr = store.get('last_ball_reset')
  return [0 if q['phase'] == 'first' else 1, q['tick1'], q['choice'], q['tick2'],
          NEVER if q['last_reset'] == -float('inf') else q['last_reset'], q['trials_left'],
          sum(1 << k for k, b in enumerate(q['pairings']) if b == 'top'), p['ttr'],
          1 if store.get('programming_complete') else 0,
          {None: 0, 'top': 1, 'bottom': 2}[store.get('which_ball')],
          NEVER if lbr is None or lbr == -float('inf') else lbr]


# ----------------------------------------------------------------------- Sequence Recall --

# (name, art ('ref' or (rows, cols) for levels.sequence_recall_art), make_game args, seed, T,
#  policy kwargs)
SEQUENCE_RECALL_CASES = (
    ('sequence_recall_paper', 'ref', (4, 60, 30, 1, 1000), 0, 1500, dict(wrong=0.15)),
    ('sequence_recall_short', 'ref', (3, 2, 1, 0, -1), 1, 500, dict(wrong=0.3)),
    ('sequence_recall_timeout', 'ref', (4, 3, 2, 2, 40), 2, 300, dict(idle_from=0)),
    ('sequence_recall_quit', 'ref', (2, 2, 2, 1, -1), 3, 300, dict(quits=((20, 0), (75, 6), (140, 0)))),
    ('sequence_recall_len1', 'ref', (1, 1, 1, 1, -1), 4, 200, dict(wrong=0.3)),
    ('sequence_recall_len16', 'ref', (16, 1, 2, 0, -1), 5, 900, dict(wrong=0.1)),
    ('sequence_recall_shape9x13', (9, 13), (5, 2, 1, 3, 120), 6, 600, dict(wrong=0.2)),
)


def _state_name(state):
  return state if isinstance(state, str) else state.name


def sequence_recall_policy(rs, centre, wrong=0.0, noise=0.03, idle_from=None, quits=()):
  """A scripted solver: in a SEEK state it walks back to `centre` and then straight toward
  the pad of the wanted light ('2' north, '4' south, '1' west, '3' east); in an EXIT state
  it steps back toward the centre.  With probability `wrong` it heads for another pad;
  `noise` is the chance of a random action; from step `idle_from` on it stands still (for
  timeouts); `quits` holds (step, action) quits."""
  heading = {'2': 1, '4': 2, '1': 3, '3': 4}
  count = [0]
  plan = {}

  def act(env):
    count[0] += 1
    for step, action in quits:
      if count[0] == step:
        return action
    if idle_from is not None and count[0] >= idle_from:
      return 5
    if rs.random_sample() < noise:
      return int(rs.randint(1, 6))
    program = env.the_plot['program'] if hasattr(env, 'the_plot') else env.plot.store['program']
    state = program[0]
    pos = tuple(env.things['P'].position)
    name = _state_name(state[0])
    if name == 'SEEK':
      key = (len(program), state[1])
      if key not in plan and pos != tuple(centre):
        return 1 if pos[0] > centre[0] else 2 if pos[0] < centre[0] else (
            3 if pos[1] > centre[1] else 4)
      if key not in plan:
        light = state[1]
        if rs.random_sample() < wrong:
          light = str(rs.choice([g for g in '1234' if g != state[1]]))
        plan[key] = heading[light]
      return plan[key]
    if name == 'EXIT':
      return 1 if pos[0] > centre[0] else 2 if pos[0] < centre[0] else (
          3 if pos[1] > centre[1] else 4)
    return 5
  return act


def sequence_recall_state(env):
  """[states left in the program, frames_in_state, timeout_frames (NO_TIMEOUT = inf)]."""
  plot = env.the_plot if hasattr(env, 'the_plot') else env.plot.store
  t = plot['timeout_frames']
  return [len(plot['program']), plot['frames_in_state'], NO_TIMEOUT if t == float('inf') else t]


# ----------------------------------------------------------------------------- running --

def closed_loop(make_env, policy, T):
  """T actions, each chosen by policy(env) before the step, on envs from make_env() under the
  auto-reset rule of tests/trajectory.py; a restart step stores 5."""
  env = make_env()
  env.its_showtime()
  actions = []
  for _ in range(T):
    if env.game_over:
      actions.append(5)
      env = make_env()
      env.its_showtime()
    else:
      actions.append(policy(env))
      env.play(actions[-1])
  return actions
