"""GPU parity of the aperture program (SURVEY.md §8f-4: two update groups, a
Drape with logic, ray casting, teleports) against the oracle.  The facade's replays of
its goldens are in test_gpu_example_goldens.py."""

import numpy as np
import pytest

import golden_cases as gc
import trajectory as tj
from oracle import games as ogames
from oracle import sampled_check

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize('which', ['aperture_stock_L1', 'aperture_stock_L2', 'other'])
def test_batched_aperture_vs_oracle(which):
  from pycolab_b200 import batched, levels
  from pycolab_b200.games import aperture
  art = levels.aperture_level() if which == 'other' else tj.u8_to_art(gc.load(which)['art'])
  B, T = 96, 400
  eng = batched.BatchedEngine([aperture.make_game(art)], batch=B)
  eng.its_showtime()
  rs = np.random.RandomState(11)
  actions = rs.choice(list(range(10)), size=(T, B),
                      p=[.14, .14, .14, .14, .04, .1, .1, .1, .095, .005]).astype(np.int32)
  last = {}
  count = {'episodes': 0, 'teleports': 0}

  def count_episodes_and_teleports(t, eng, worlds, outs):
    for e, w in worlds.items():
      now = w.things['A'].position
      if e in last and last[e][0] is not w:   # the world was rebuilt: an episode ended
        count['episodes'] += 1
      elif e in last:
        before = last[e][1]
        count['teleports'] += abs(before[0] - now[0]) + abs(before[1] - now[1]) > 1
      last[e] = (w, now)
  sampled_check.lockstep(eng, lambda e: ogames.make_aperture(art), range(B), actions,
                         curtains='X', sprites='A', on_step=count_episodes_and_teleports)
  assert count['episodes'] > 0 and count['teleports'] > 0
  assert int(eng.error_codes().abs().max()) == 0
