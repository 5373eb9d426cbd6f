"""`Scrolly` (reference `pycolab/prefab_parts/drapes.py:30-695`).

Set-up side of the Scrolly prefab: the constructor contract (board shape,
whole pattern, north-west corner, margins, scrolling group) with the same
validation, the initial curtain, and `PatternInfo` for ASCII-art worlds.  The
per-step half — `_maybe_move` (drapes.py:487-659) and the
`pattern_position_*` look-ups — is `pcl::scrolly_move` /
`pcl::scrolly_touch_prescroll` in csrc/pcl_device.cuh; on the device the
pattern is bit-packed and the curtain is a window into it that is never
stored.
"""

import numpy as np

from pycolab_b200 import ascii_art
from pycolab_b200 import things
from pycolab_b200.errors import DeviceOnlyError


class Scrolly(things.Drape):
  """A drape whose curtain is a board-sized window onto a larger pattern."""

  _NORTH, _NORTHEAST, _EAST, _SOUTHEAST = (-1, 0), (-1, 1), (0, 1), (1, 1)
  _SOUTH, _SOUTHWEST, _WEST, _NORTHWEST = (1, 0), (1, -1), (0, -1), (-1, -1)
  _STAY = (0, 0)

  class PatternInfo(object):
    """Interpret an ASCII-art world for Scrolly constructors (drapes.py:166-291)."""

    def __init__(self, whole_pattern_art, board_art_or_shape,
                 board_northwest_corner_mark, what_lies_beneath):
      if ord(what_lies_beneath) > 127:
        raise ValueError('The what_lies_beneath value used to build a '
                         'Scrolly.PatternInfo must be an ASCII character.')
      self._art = ascii_art.ascii_art_to_uint8_nparray(whole_pattern_art)
      self._corner = self._find(board_northwest_corner_mark,
                                'the Scrolly.PatternInfo constructor')
      self._art[self._corner] = ord(what_lies_beneath)
      try:
        self._board_shape = (len(board_art_or_shape), len(board_art_or_shape[0]))
      except TypeError:
        rows, cols = board_art_or_shape
        self._board_shape = (rows, cols)
      if (self._board_shape[0] > self._art.shape[0] or
          self._board_shape[1] > self._art.shape[1]):
        raise ValueError(
            'The whole_pattern_art value used to build a Scrolly.PatternInfo (size '
            '{}) cannot completely cover the game board (size {}).'.format(
                self._art.shape, self._board_shape))

    def virtual_position(self, character):
      where = self._find(character, 'Scrolly.PatternInfo.virtual_position()')
      return (where[0] - self._corner[0], where[1] - self._corner[1])

    def kwargs(self, character):
      return {'board_shape': self._board_shape,
              'whole_pattern': self._art == ord(character),
              'board_northwest_corner': self._corner}

    def _find(self, character, who):
      hits = np.argwhere(self._art == ord(character))
      if len(hits) == 0:
        raise RuntimeError('{} found no instances of {!r} in the pattern art used to '
                           'build this PatternInfo object.'.format(who, character))
      if len(hits) > 1:
        raise RuntimeError('{} found multiple instances of {!r} in the pattern art '
                           'used to build this PatternInfo object.'.format(
                               who, character))
      return (int(hits[0][0]), int(hits[0][1]))

  def __init__(self, curtain, character, board_shape, whole_pattern,
               board_northwest_corner, scroll_margins=(2, 3), scrolling_group=''):
    super(Scrolly, self).__init__(curtain, character)
    self._board_shape = tuple(board_shape)
    self._northwest_corner = things.Sprite.Position(*board_northwest_corner)
    self._scrolling_group = scrolling_group
    self._w_h_o_l_e_p_a_t_t_e_r_n = whole_pattern
    # The pattern as handed in, before a subclass's constructor edits it (t_maze.py:365
    # speckles it at random): a device that redraws at every restart starts from this.
    self._pattern_at_init = np.array(whole_pattern, dtype=bool)
    self._northwest_corner_limit = (whole_pattern.shape[0] - board_shape[0],
                                    whole_pattern.shape[1] - board_shape[1])
    if min(self._northwest_corner_limit) < 0:
      raise ValueError(
          'The whole_pattern provided to the `Scrolly` constructor (size {}) cannot '
          'completely cover the game board (size {}).'.format(
              whole_pattern.shape, board_shape))
    self._have_margins = scroll_margins is not None
    self._scroll_margins = None if scroll_margins is None else tuple(scroll_margins)
    if self._have_margins:
      self._margin_north = scroll_margins[0] - 1
      self._margin_south = board_shape[0] - scroll_margins[0]
      self._margin_west = scroll_margins[1] - 1
      self._margin_east = board_shape[1] - scroll_margins[1]
      if (self._margin_west >= self._margin_east or
          self._margin_north >= self._margin_south):
        raise ValueError(
            'The scrolling margins provided to the `Scrolly` constructor, {}, are so '
            'large that a margin would overlap more than half of the '
            'board.'.format(scroll_margins))
    self._update_curtain()
    self._last_maybe_move_frame = -float('inf')
    self._prescroll_northwest_corner = self._northwest_corner

  @property
  def whole_pattern(self):
    return self._w_h_o_l_e_p_a_t_t_e_r_n

  def pattern_position_prescroll(self, virtual_position, the_plot):
    if self._last_maybe_move_frame < the_plot.frame:
      self._prescroll_northwest_corner = self._northwest_corner
    return things.Sprite.Position(
        virtual_position[0] + self._prescroll_northwest_corner[0],
        virtual_position[1] + self._prescroll_northwest_corner[1])

  def pattern_position_postscroll(self, virtual_position, the_plot):
    if self._last_maybe_move_frame < the_plot.frame:
      raise RuntimeError(
          'The pattern_position_postscroll method was called on a Scrolly instance '
          'before that instance had a chance to decide whether or where it would '
          'scroll.')
    return things.Sprite.Position(virtual_position[0] + self._northwest_corner[0],
                                  virtual_position[1] + self._northwest_corner[1])

  def _update_curtain(self):
    r, c = self._northwest_corner
    np.copyto(self.curtain, self.whole_pattern[r:r + self._board_shape[0],
                                               c:c + self._board_shape[1]])

  def _device_only(self, *unused_args, **unused_kwargs):
    raise DeviceOnlyError(
        'Scrolly motion helpers run inside the CUDA step kernel '
        '(pcl::scrolly_move); pycolab_b200 never executes update() in Python.')

  _northwest = _north = _northeast = _east = _southeast = _device_only
  _south = _southwest = _west = _stay = _device_only
