"""Generate the Cued Catch and Sequence Recall golden fixtures (tests/golden/cued_catch_*.npz,
tests/golden/sequence_recall_*.npz) from the UNMODIFIED reference.

Run in the build container (where /root/reference exists):

    python tests/golden/make_lp_rnn_golden.py

Neither reference file runs on Python 3 with NumPy 2 as it is; the two shims of
tests/lp_rnn_cases.py (Python 2's None ordering for Cued Catch, NumPy 1's boolean `-=` for
Sequence Recall) act on the built Engine and patch no source.  Each file holds the art, the
make_game arguments and seed (JSON), the closed-loop policy's actions and what the reference
produced for them: board per frame, the float64 reward and its Python type, discount,
game_over, the sprites and the game's private state of every frame.
"""

import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from make_golden import refdriver, save, tj  # noqa: E402
import lp_rnn_cases as lc                                      # noqa: E402

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


def small_cued_catch_art():
  """5 x 14: a width that is no multiple of 4, 'Q' cells in row 0, balls in other columns,
  and fewer than 7 rows, so the bands 3:5 and -2: overlap."""
  from pycolab_b200 import levels
  return levels.cued_catch_art(5, 14, player=(1, 2), balls=((1, 9), (2, 12)),
                               cue_cells=((0, 0), (0, 5), (0, 13), (2, 7)))


def cued_catch():
  import random
  ref = lc.ref_module('cued_catch')
  for name, art, args, seed, T, kw in CUED_CATCH_CASES:
    art = list(ref.GAME_ART) if art is None else small_cued_catch_art()
    sprites, rewards, types, states = [], [], [], []

    def on_frame(env, out):
      sprites.append(tj.sprite_rows(env, 'Pab'))
      rewards.append(np.nan if out[1] is None else float(out[1]))
      types.append(lc.reward_code(out[1]))
      states.append(lc.cued_catch_state(env))
    random.seed(900 + seed)
    make = lambda: lc.shim_cued_catch(lc.with_art(ref, art, lambda: ref.make_game(*args)))
    policy = lc.cued_catch_policy(np.random.RandomState(seed), **kw)
    traj, actions = lc.closed_loop(make, policy, T, on_frame=on_frame)
    config = dict(args=list(args), seed=900 + seed)
    save(name, art=tj.art_to_u8(art), actions=np.array(actions, dtype=np.int32),
         sprites=np.array(sprites, dtype=np.int32),
         reward_f64=np.array(rewards, dtype=np.float64), reward_type=np.array(types, np.uint8),
         state=np.array(states, dtype=np.int64),
         config=np.frombuffer(json.dumps(config).encode(), dtype=np.uint8), **traj)
    r = np.array(rewards)
    print('  %s: %d episodes, reward sum %.3f, float frames %d' % (
        name, int(traj['game_over'].sum()), float(np.nansum(r)), int((np.array(types) == 2).sum())))


def sequence_recall():
  import random
  from pycolab_b200 import levels
  ref = lc.ref_module('sequence_recall')
  for name, art, args, seed, T, kw in SEQUENCE_RECALL_CASES:
    art = list(ref.GAME_ART) if art == 'ref' else levels.sequence_recall_art(*art)
    centre = tuple(int(x[0]) for x in np.where(tj.art_to_u8(art) == ord('P')))
    sprites, rewards, states = [], [], []

    def on_frame(env, out):
      sprites.append(tj.sprite_rows(env, 'P'))
      rewards.append(np.nan if out[1] is None else float(out[1]))
      states.append(lc.sequence_recall_state(env))
    random.seed(900 + seed)
    make = lambda: lc.shim_sequence_recall(lc.with_art(ref, art, lambda: ref.make_game(*args)))
    policy = lc.sequence_recall_policy(np.random.RandomState(seed), centre, **kw)
    traj, actions = lc.closed_loop(make, policy, T, on_frame=on_frame)
    config = dict(args=list(args), seed=900 + seed)
    save(name, art=tj.art_to_u8(art), actions=np.array(actions, dtype=np.int32),
         sprites=np.array(sprites, dtype=np.int32),
         reward_f64=np.array(rewards, dtype=np.float64), state=np.array(states, dtype=np.int64),
         config=np.frombuffer(json.dumps(config).encode(), dtype=np.uint8), **traj)
    r = np.array(rewards)
    print('  %s: %d episodes, +1 %d, wrong %d' % (
        name, int(traj['game_over'].sum()), int((r > 0.9).sum()),
        int((r == -0.005).sum() - 0)))


if __name__ == '__main__':
  assert refdriver.available(), '/root/reference is required'
  cued_catch()
  sequence_recall()
