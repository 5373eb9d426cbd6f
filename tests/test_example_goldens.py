"""The oracle (oracle/games.py, and the chained worlds of the Ordeal) replays every
example-game golden of tests/example_games.py REPLAYS: every array the golden
holds, frame by frame, boards, rewards, sprite registers, curtains, croppers' views and
corners, chapters and float registers included.
"""

import pytest

import example_games as eg


@pytest.mark.parametrize('name', eg.REPLAYS)
def test_oracle_replays(name):
  eg.assert_replays('oracle', name)
