"""GPU parity of the better_scrolly_maze program (SURVEY.md §8f-1) and its three
cropper views, against the oracle.  The facade's replays of its goldens are in
test_gpu_example_goldens.py."""

import numpy as np
import pytest

import golden_cases as gc
import trajectory as tj
from oracle import engine_model as em
from oracle import games as ogames
from oracle import sampled_check

pytestmark = pytest.mark.gpu


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
