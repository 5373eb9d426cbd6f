"""`storytelling.Story` over device-backed Engines (and device croppers) against
the golden trajectories the reference's Story produced (SURVEY.md §8f-4)."""

import pytest

import example_games as eg

pytestmark = pytest.mark.gpu


def test_list_story_of_device_games():
  eg.assert_replays('facade', 'story_classics_list')


def test_dict_story_with_device_croppers():
  eg.assert_replays('facade', 'story_classics_cropped')
