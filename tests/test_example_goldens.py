"""The oracle (oracle/games.py, the research games' oracles, and the chained worlds of the
Ordeal) replays every golden of tests/example_games.py REPLAYS: every array the golden holds,
frame by frame, boards, rewards, sprite registers, curtains, croppers' views and corners,
chapters, float registers and the research games' private state included.
"""

import pytest

import example_games as eg


@pytest.mark.parametrize('name', eg.REPLAYS)
def test_oracle_replays(name):
  eg.assert_replays('oracle', name)
