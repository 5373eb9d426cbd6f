"""The oracle interpreter (oracle/compiled.py) running the compiled words of every
registered-game module (tests/registered_games.py MODULES) reproduces each golden the
reference made of it: every array the golden holds, frame by frame, registers, Plot keys,
Scrolly corners and patterns, Backdrop curtains and the global generators' final words
included.  Where the reference raised, the oracle raises IndexError as it did, and latches
PCL_ENV_ERR_ARITH for a ZeroDivisionError, as the device does.
"""

import pytest

import registered_games as rg


@pytest.fixture(scope='module')
def games(request):
  yield from rg.registered(request.param)


@pytest.mark.parametrize('games,name', rg.GOLDENS, indirect=['games'],
                         ids=[name for _, name in rg.GOLDENS])
def test_oracle_replays_registered_golden(games, name):
  rg.assert_oracle_replays(games, name)
