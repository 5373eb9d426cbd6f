"""GPU parity of the better_scrolly_maze program (SURVEY.md §8f-1) and its three
cropper views, against the reference's golden trajectories and the oracle."""

import numpy as np
import pytest

import golden_cases as gc
import trajectory as tj
from oracle import engine_model as em
from oracle import games as ogames
from oracle import sampled_check

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize('name', gc.names('better_'))
def test_facade_better_scrolly_golden_with_croppers(name):
  from pycolab_b200.games import better_scrolly_maze as bsm
  g = gc.load(name)
  art = tj.u8_to_art(g['art'])
  croppers = bsm.make_croppers(tuple(int(x) for x in g['starter_offset']),
                               tuple(int(x) for x in g['teaser_corner']))
  sprites, views = [], [[], [], []]
  n = min(len(g['actions']), 250)

  def make():
    eng = bsm.make_game(art)
    for c in croppers:
      c.set_engine(eng)
    return eng

  def on_frame(env, out):
    rows = []
    for ch in 'Pabc':
      s = env.things[ch]
      rows.append([s.position[0], s.position[1], int(bool(s.visible)),
                   s.virtual_position[0], s.virtual_position[1]])
    sprites.append(rows)
    for v, c in zip(views, croppers):
      v.append(c.crop(out[0]).board)

  got = tj.run_trajectory(make, g['actions'][:n].tolist(), on_frame=on_frame)
  want = {k: g[k][:n + 1] for k in ('boards', 'reward', 'has_reward', 'discount',
                                    'game_over')}
  tj.assert_same_trajectory(want, got, name)
  np.testing.assert_array_equal(g['sprites'][:n + 1], np.array(sprites))
  for key, v in zip(('view_player', 'view_patroller', 'view_teaser'), views):
    np.testing.assert_array_equal(g[key][:n + 1], np.stack(v), err_msg=key)


def test_batched_better_scrolly_vs_oracle():
  from pycolab_b200 import batched
  from pycolab_b200.games import better_scrolly_maze as bsm
  g = gc.load('better_stock_L1')
  art = tj.u8_to_art(g['art'])
  B, T = 20, 300
  eng = batched.BatchedEngine([bsm.make_game(art)], batch=B)
  eng.its_showtime()
  rs = np.random.RandomState(8)
  actions = rs.randint(0, 6, size=(T, B)).astype(np.int32)
  actions[rs.random_sample(actions.shape) < 0.97] %= 5
  spec = batched.scrolling_crop_spec(7, 10, eng.sprite_chars.index('c'), pad_char=' ',
                                     scroll_margins=(None, 3))
  sampled_check.lockstep(
      eng, lambda e: ogames.make_better_scrolly(art), range(B), actions, curtains='@',
      crop=(spec, None, lambda: em.ScrollingCrop(7, 10, ['c'], pad_char=' ',
                                                 scroll_margins=(None, 3))))
  assert int(eng.error_codes().abs().max()) == 0
