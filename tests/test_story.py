"""`storytelling.Story` (host-side caller of the path) on CPU.

The Story logic is driven here by oracle Worlds dressed as Engines (OracleEngine),
against the golden trajectory the reference's own Story produced for the same chapters
(tests/golden/story_classics_list.npz); plus the constructor's argument checks
(storytelling.py:493-622).
"""

import numpy as np
import pytest

import example_games as eg
import story_cases
from story_cases import OracleEngine, oracle_chapter
from oracle import games as ogames
from pycolab_b200 import storytelling
from pycolab_b200 import things


def test_list_story_matches_reference_golden():
  eg.assert_replays('oracle', 'story_classics_list')


def test_story_views_and_plot_hand_over():
  story = storytelling.Story([oracle_chapter(k, a) for k, a in story_cases.LIST_CHAPTERS])
  story.its_showtime()
  assert (story.rows, story.cols) == (4, 12)
  assert story.z_order == ['P'] and set(story.backdrop.palette) == {'.'}
  assert not storytelling.is_fictional(story.things['P'])
  story.the_plot['note'] = 42
  first = story.current_game
  # one step east falls off the cliff: chapter 0 ends, chapter 1 starts in the same call
  obs, reward, discount = story.play(3)
  assert first.game_over and story.current_game is not first and not story.game_over
  assert story.the_plot['note'] == 42                       # Plot entries travel
  assert (story.the_plot.prior_chapter, story.the_plot.this_chapter,
          story.the_plot.next_chapter) == (0, 1, 2)
  assert reward == -100.0 and discount == 1.0               # new game's discount, old reward
  with pytest.raises(RuntimeError):
    story.its_showtime()


def test_story_ends_after_last_chapter_and_refuses_more_play():
  story = storytelling.Story([oracle_chapter('chain_walk', None)])
  story.its_showtime()
  for _ in range(2):
    obs, reward, discount = story.play(0)
  assert story.game_over and reward == 1.0 and discount == 0.0
  with pytest.raises(RuntimeError):
    story.play(0)


def test_dict_story_follows_next_chapter_and_rejects_unknown_keys():
  def cliff_then(target):
    def build():
      game = oracle_chapter('cliff_walk', None)()
      game.the_plot.next_chapter = target
      return game
    return build
  story = storytelling.Story({'a': cliff_then('b'), 'b': cliff_then(None)}, first_chapter='a')
  story.its_showtime()
  story.play(3)
  assert story.the_plot.this_chapter == 'b' and story.the_plot.prior_chapter == 'a'
  bad = storytelling.Story({'a': cliff_then('nowhere')}, first_chapter='a')
  bad.its_showtime()
  with pytest.raises(KeyError):
    bad.play(3)


def test_constructor_argument_checks():
  rooms, cliff = oracle_chapter('four_rooms', None), oracle_chapter('cliff_walk', None)
  with pytest.raises(ValueError):
    storytelling.Story([])
  with pytest.raises(ValueError):
    storytelling.Story({None: cliff}, first_chapter=None)
  with pytest.raises(ValueError):
    storytelling.Story({'a': cliff}, first_chapter='b')
  with pytest.raises(ValueError):
    storytelling.Story([cliff, cliff], croppers=[None])          # keys differ
  with pytest.raises(ValueError):
    storytelling.Story([rooms, cliff])                           # 13x13 vs 4x12 observations

  class _DrapeP(OracleEngine):                                   # 'P' as a Drape elsewhere
    @property
    def things(self):
      class D(things.Drape):
        def update(self, *args, **kwargs):
          pass
      return {'P': D(np.zeros((self.rows, self.cols), dtype=bool), 'P')}
  clash = lambda: _DrapeP(ogames.make_classic('cliff_walk', ['............'] * 3 + ['P...........']), '.')
  with pytest.raises(ValueError):
    storytelling.Story([cliff, clash])


def test_reference_story_tests_pass_against_this_story_class(monkeypatch):
  """The reference's own `tests/story_test.py` (6 tests: sequences, dicts,
  cropping, inter-game reward accumulation, stand-ins, compatibility checking),
  UNMODIFIED, with `storytelling.Story` replaced by this package's class.  The
  chapters are reference Engines (the tests define entities with Python update
  logic), so the class is pointed at the reference's `things` / `cropping` /
  `engine` types for the duration."""
  import sys
  import unittest
  import refdriver
  if not refdriver.available():
    pytest.skip('/root/reference not present')
  refdriver.ref_storytelling()          # the Python 3.12 collections shim + import path
  from pycolab import cropping as ref_cropping
  from pycolab import engine as ref_engine
  from pycolab import things as ref_things
  from pycolab.tests import story_test
  monkeypatch.setattr(storytelling, 'cropping', ref_cropping)
  monkeypatch.setattr(storytelling, 'things', ref_things)
  monkeypatch.setattr(storytelling, 'engine_lib', ref_engine)
  monkeypatch.setattr(story_test, 'storytelling', storytelling)
  suite = unittest.defaultTestLoader.loadTestsFromModule(story_test)
  result = unittest.TextTestRunner(verbosity=0).run(suite)
  assert result.testsRun == 6 and result.wasSuccessful(), result.failures + result.errors
