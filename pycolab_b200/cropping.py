"""Observation croppers (reference `pycolab/cropping.py:27-598`).

Same classes and constructor arguments.  `crop()` runs on the device
(`pcl_crop`, csrc/render.cu `crop_kernel`): the window corner of a
`ScrollingCropper` is per-env device state next to the plot record, so in a
`BatchedEngine` every env pans/saccades its own window; this facade drives the
batch-1 engine behind a `pycolab_b200.engine.Engine`.
"""

import copy

import numpy as np

from pycolab_b200 import rendering
from pycolab_b200.errors import NotLoweredError


class ObservationCropper(object):
  """Identity cropper / base class (cropping.py:27-227)."""

  def __init__(self):
    self._engine = None
    self._pad_char = None

  def set_engine(self, engine):
    if engine is not self._engine:
      self._state = None          # a new Engine forgets the window (cropping.py:375-391)
    self._engine = engine

  def crop(self, observation):
    return observation

  @property
  def rows(self):
    return self._engine.rows

  @property
  def cols(self):
    return self._engine.cols

  def _check_pad(self):
    if self._pad_char is not None:
      legal = set(self._engine.things) | set(self._engine.backdrop.palette)
      if self._pad_char not in legal:
        raise ValueError("An `ObservationCropper` tried to fill empty space with a "
                         "character that isn't used by the current game engine.")

  def _device_crop(self, spec, observation):
    self._check_pad()
    b = self._engine.batched
    if b is None:
      raise RuntimeError('crop() called before the Engine entered play mode')
    if getattr(self, '_state', None) is None:
      self._state = b.new_crop_state()
    board = b.crop(spec, state=self._state)[0].cpu().numpy().copy()
    layers = getattr(observation, 'layers', None)
    if layers is None or isinstance(layers, rendering.LazyLayers):
      # occluded layers: those of the cropped board, pad cells included
      chars = set(self._engine.things) | set(self._engine.backdrop.palette)
      return rendering.Observation(board=board, layers=rendering.LazyLayers(board, chars))
    # Un-occluded layers (occlusion_in_layers=False) are not a function of the board:
    # crop each as _do_crop does (cropping.py:189-219), at the corner the device chose.
    if spec.sprite_index < 0:
      corner = (spec.offset_rows, spec.offset_cols)
    else:
      corner = tuple(int(v) for v in self._state[0, :2].cpu())
    return rendering.Observation(board=board, layers=crop_layers(
        layers, corner, spec.rows, spec.cols, self._pad_char))


def crop_layers(layers, corner, rows, cols, pad_char):
  """`_do_crop`'s layer part (cropping.py:189-219): each layer's rows x cols window at
  `corner`, cells off the board set where the layer's character is `pad_char`."""
  top, left = corner
  out = {}
  for char, layer in layers.items():
    H, W = layer.shape
    got = np.full((rows, cols), pad_char == char, dtype=bool)
    r0, c0 = max(0, top), max(0, left)
    r1, c1 = max(0, min(H, top + rows)), max(0, min(W, left + cols))
    if r1 > r0 and c1 > c0:
      got[r0 - top:r1 - top, c0 - left:c1 - left] = layer[r0:r1, c0:c1]
    out[char] = got
  return out


class FixedCropper(ObservationCropper):
  """A fixed window, optionally padded (cropping.py:229-310)."""

  def __init__(self, top_left_corner, rows, cols, pad_char=None):
    super(FixedCropper, self).__init__()
    self._top_row, self._left_col = top_left_corner
    self._rows, self._cols = rows, cols
    self._pad_char = pad_char

  def crop(self, observation):
    from pycolab_b200 import _lib
    if self._pad_char is None and (
        self._top_row < 0 or self._left_col < 0 or
        self._top_row + self._rows > self._engine.rows or
        self._left_col + self._cols > self._engine.cols):
      raise RuntimeError('An ObservationCropper attempted to crop a region that extends '
                         'beyond the observation without specifying a character to fill '
                         'the void that exists out there.')
    spec = _lib.CropSpec(self._rows, self._cols, -1,
                         -1 if self._pad_char is None else ord(self._pad_char),
                         0, 0, self._top_row, self._left_col, 0)
    return self._device_crop(spec, observation)

  @property
  def rows(self):
    return self._rows

  @property
  def cols(self):
    return self._cols


class ScrollingCropper(ObservationCropper):
  """A window that follows an entity (cropping.py:313-598)."""

  def __init__(self, rows, cols, to_track, pad_char=None, scroll_margins=(2, 3),
               initial_offset=None, saccade=True):
    super(ScrollingCropper, self).__init__()
    from pycolab_b200 import batched
    self._rows, self._cols = rows, cols
    self._to_track = copy.copy(to_track)
    self._pad_char = pad_char
    # Validates and resolves margins exactly as cropping.py:362-380.
    self._spec_args = dict(pad_char=pad_char, scroll_margins=scroll_margins,
                           initial_offset=initial_offset, saccade=saccade)
    batched.scrolling_crop_spec(rows, cols, 0, **self._spec_args)

  def set_engine(self, engine):
    prior = self._engine
    super(ScrollingCropper, self).set_engine(engine)
    if engine is not prior:
      if ((engine.rows < self._rows or engine.cols < self._cols) and
          self._pad_char is None):
        raise ValueError(
            "A ScrollingCropper with a size of {} and no pad character can't be used "
            'with a pycolab engine that produces smaller observations in any dimension '
            '(in this case, {})'.format((self._rows, self._cols),
                                        (engine.rows, engine.cols)))

  def crop(self, observation):
    from pycolab_b200 import batched
    from pycolab_b200 import _lib
    b = self._engine.batched
    if b is None:
      raise RuntimeError('crop() called before the Engine entered play mode')
    if not 0 < len(self._to_track) <= _lib.MAX_TRACK:
      raise NotLoweredError('the device cropper tracks 1..{} entities'.format(_lib.MAX_TRACK))
    codes = []                     # priority list: k > 0 sprite k - 1, k < 0 drape -k - 1
    for char in self._to_track:
      if char not in self._engine.things:
        raise RuntimeError('ScrollingCropper was told to track a nonexistent game entity '
                           '{!r}.'.format(char))
      if char in b.sprite_chars:
        codes.append(b.sprite_chars.index(char) + 1)
      elif char in b.drape_chars:
        codes.append(-(b.drape_chars.index(char) + 1))
      else:                      # e.g. a box_world key: an object of the program, no drape
        raise NotLoweredError('the device cropper tracks sprites and drapes only; {!r} is '
                              'neither in this game'.format(char))
    spec = batched.scrolling_crop_spec(self._rows, self._cols, 0, track=codes,
                                       **self._spec_args)
    return self._device_crop(spec, observation)

  @property
  def rows(self):
    return self._rows

  @property
  def cols(self):
    return self._cols
