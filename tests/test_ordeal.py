"""examples/ordeal.py (SURVEY.md §8f-4): a `storytelling.Story` of three sub-games
whose entities carry `has_sword` / `last_position` across chapters in the Plot and
issue `Plot.change_z_order` on a real game (ordeal.py:182-185).

Goldens (tests/golden/ordeal_*.npz) are the reference's own Story on BFS-scripted
walks (sword + victory, no sword + defeat, castle and back, quit) and random walks,
replayed in test_example_goldens.py (the oracle restatement chained like Story does,
example_games.OracleOrdeal) and test_gpu_example_goldens.py (this package's Story over
device-backed Engines and the device cropper).  Here: what the goldens cover, the
battle's z-order on the device and, where the reference is installed, its unmodified
ordeal.py loaded through `compat` lowering to the same device state.
"""

import os

import numpy as np
import pytest

import golden_cases as gc
import refdriver


def test_goldens_cover_the_interesting_paths():
  wins, loses = gc.load('ordeal_sword_wins'), gc.load('ordeal_no_sword_loses')
  assert wins['reward'].sum() == 2 and set(wins['chapters'].tolist()) == {'kansas', 'cavern',
                                                                          'castle'}
  assert loses['reward'].sum() == -1 and loses['has_sword'].max() == 0
  assert wins['has_sword'].max() == 1 and int(wins['game_over'].sum()) >= 1


@pytest.mark.gpu
def test_device_ordeal_z_order_follows_the_battle():
  """ordeal.py:182-185 on the device: the winner is drawn on top."""
  from pycolab_b200.games import ordeal
  for name, front in (('ordeal_sword_wins', 'D'), ('ordeal_no_sword_loses', 'P')):
    g = gc.load(name)
    story = ordeal.make_game()
    story.its_showtime()
    for a in g['actions'].tolist():
      story.play(a)
      if story.game_over:
        break
    assert story.game_over and story.the_plot.this_chapter == 'castle'
    assert story.current_game.z_order[-1] == front, name


@pytest.mark.skipif(not refdriver.available(), reason='/root/reference not present')
def test_reference_ordeal_chapters_lower_like_the_twins():
  import sys
  from pycolab_b200 import compat, lowering
  from pycolab_b200.games import ordeal
  saved = {k: v for k, v in sys.modules.items() if k == 'pycolab' or k.startswith('pycolab.')}
  compat.uninstall()
  try:
    mod = compat.load_example(os.path.join(refdriver.REFERENCE_ROOT, 'pycolab', 'examples',
                                           'ordeal.py'))
    # the reference builds its chapters inside make_game(): rebuild them here with
    # ITS classes and art (ordeal.py:77-93)
    aa = mod.ascii_art
    theirs = {
        'castle': aa.ascii_art_to_game(mod.GAME_ART_CASTLE, what_lies_beneath=' ',
                                       sprites=dict(P=mod.PlayerSprite, D=mod.DragonduckSprite),
                                       update_schedule=['P', 'D'], z_order=['D', 'P']),
        'cavern': aa.ascii_art_to_game(mod.GAME_ART_CAVERN, what_lies_beneath=' ',
                                       sprites=dict(P=mod.PlayerSprite),
                                       drapes=dict(S=mod.SwordDrape), update_schedule=['P', 'S']),
        'kansas': aa.ascii_art_to_game(mod.GAME_ART_KANSAS, what_lies_beneath='~',
                                       sprites=dict(P=mod.PlayerSprite))}
    mine = {'castle': ordeal.make_castle(), 'cavern': ordeal.make_cavern(),
            'kansas': ordeal.make_kansas()}
    for chapter in theirs:
      a, b = lowering.lower(theirs[chapter]), lowering.lower(mine[chapter])
      assert a.signature() == b.signature(), chapter
      for field in ('backdrop', 'sprites', 'drapes', 'plot'):
        np.testing.assert_array_equal(getattr(a, field), getattr(b, field), err_msg=chapter)
      for d in a.bits:
        np.testing.assert_array_equal(a.bits[d], b.bits[d])
  finally:
    compat.uninstall()
    sys.modules.update(saved)
