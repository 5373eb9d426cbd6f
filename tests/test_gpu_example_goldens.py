"""The facade Engine on the H100 replays every example-game golden of
tests/example_games.py REPLAYS: every array the golden holds, frame by frame, up to the family's
frame limit, with the global generators seeded as the reference's were.
"""

import pytest

import example_games as eg
from registered_games import global_generators  # noqa: F401  (a fixture)

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize('name', eg.REPLAYS)
def test_facade_replays(global_generators, name):  # noqa: F811
  eg.assert_replays('facade', name)
