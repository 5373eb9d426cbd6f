"""The facade Engine on the H100 replays every golden of the registered-game modules
(tests/registered_games.py MODULES): every array the golden holds, frame by frame, with the
global generators seeded as the reference's were and continuing where its stopped.  Every
register and Plot key keeps, at every frame, the Python type it has in a freshly made game,
and where the reference raised the facade raises the same exception.
"""

import pytest

import registered_games as rg
from registered_games import global_generators  # noqa: F401  (a fixture)

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def games(request):
  yield from rg.registered(request.param)


@pytest.mark.parametrize('games,name', rg.GOLDENS, indirect=['games'],
                         ids=[name for _, name in rg.GOLDENS])
def test_facade_replays_registered_golden(games, global_generators, name):  # noqa: F811
  rg.assert_facade_replays(games, name)
