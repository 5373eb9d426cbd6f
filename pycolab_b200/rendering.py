"""Observations and the base renderer (reference `pycolab/rendering.py:28-301`).

`Observation(board, layers)` is the same namedtuple.  In occluded mode the
reference's layers are exactly `board == ord(c)` for every legal character
(rendering.py:177-178), so they are never stored or shipped: `LazyLayers`
derives a mask on first access.

`BaseObservationRenderer` keeps the reference's canvas protocol
(`clear` / `paint_all_of` / `paint_sprite` / `paint_drape` / `render`) but the
paint + occlusion flatten runs on the GPU: `render()` uploads what was painted
and launches the stand-alone render kernel through `pcl_render`
(csrc/render.cu).  The z-order is the order of the paint calls, as upstream.
"""

import collections
import ctypes as C

import numpy as np


class Observation(collections.namedtuple('Observation', ['board', 'layers'])):
  """board: uint8 [rows, cols]; layers: {char: bool [rows, cols]}.  Read-only;
  contents are only valid until the next render (rendering.py:55-63)."""
  __slots__ = ()


class LazyLayers(collections.abc.Mapping):
  """{char: board == ord(char)} computed on demand (rendering.py:177-178)."""

  def __init__(self, board, chars):
    self._board = board
    self._chars = frozenset(chars)
    self._cache = {}

  @property
  def board(self):
    """The board these layers are derived from."""
    return self._board

  def __getitem__(self, char):
    if char not in self._chars:
      raise KeyError(char)
    if char not in self._cache:
      self._cache[char] = self._board == ord(char)
    return self._cache[char]

  def __iter__(self):
    return iter(self._chars)

  def __len__(self):
    return len(self._chars)


class BaseObservationRenderer(object):
  """GPU-backed canvas with the reference's painter API (rendering.py:69-184)."""

  def __init__(self, rows, cols, characters):
    self._rows, self._cols = rows, cols
    self._chars = set(characters)
    self._backdrop = np.zeros((rows, cols), dtype=np.uint8)
    self._painted = []            # (kind, char, data) in paint (= z) order
    self._handles = {}

  def clear(self):
    self._backdrop = np.zeros((self._rows, self._cols), dtype=np.uint8)
    self._painted = []

  def paint_all_of(self, curtain):
    curtain = np.asarray(curtain)
    if curtain.dtype != np.uint8 or curtain.shape != (self._rows, self._cols):
      raise TypeError('paint_all_of needs a uint8 array shaped like the canvas')
    self._backdrop = curtain.copy()
    self._painted = []            # copies over everything painted so far

  def paint_sprite(self, character, position):
    self._check(character)
    row, col = int(position[0]), int(position[1])
    # `self._board[tuple(position)]` upstream: NumPy wraps a negative index once
    # and raises beyond that.
    if not (-self._rows <= row < self._rows and -self._cols <= col < self._cols):
      raise IndexError('sprite position {} is off the {}x{} board'.format(
          (row, col), self._rows, self._cols))
    self._painted.append(('sprite', character, (row, col)))

  def paint_drape(self, character, curtain):
    self._check(character)
    self._painted.append(('drape', character, np.asarray(curtain, dtype=bool).copy()))

  def _check(self, character):
    if character not in self._chars:
      raise ValueError('character {} does not seem to be a valid character for this '
                       'game'.format(str(character)))

  def render(self):
    board = render_on_device(self._backdrop, self._painted)
    return Observation(board=board, layers=LazyLayers(board, self._chars))

  @property
  def shape(self):
    return (self._rows, self._cols)


class _BoardOnDevice(object):
  """A batch-1 handle (no step program) to run pcl_observe over one board."""

  def __init__(self):
    self._handles = {}

  def __call__(self, board, table, valid, is_3d, permute, want_unknown=False):
    import torch
    from pycolab_b200 import _lib
    from pycolab_b200 import observers
    lib = _lib.load()
    rows, cols = board.shape
    pitch = (cols + 15) // 16 * 16
    key = (rows, cols)
    if key not in self._handles:
      spec = _lib.Spec()
      spec.abi_version, spec.program = _lib.ABI_VERSION, _lib.PROG_NONE
      spec.rows, spec.cols, spec.pitch = rows, cols, pitch
      handle = C.c_void_p()
      _lib.check(lib.pcl_create(C.byref(spec), 1, 0, C.byref(handle)), 'pcl_create')
      self._handles[key] = handle
    dev = torch.device('cuda', 0)
    padded = np.zeros((1, rows, pitch), dtype=np.uint8)
    padded[0, :, :cols] = board
    t_board = torch.from_numpy(padded).to(dev)
    unknown = torch.zeros((1,), dtype=torch.int32, device=dev) if want_unknown else None
    stream = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    out = observers.observe(lib, self._handles[key], t_board, rows, cols, table, valid,
                            is_3d, permute, stream, unknown)
    torch.cuda.synchronize(dev)
    return (observers.numpy_view(out[0], table.dtype),
            bool(int(unknown[0])) if want_unknown else False)


_on_device = _BoardOnDevice()


class ObservationToArray(object):
  """Characters -> scalars or vectors (rendering.py:409-542); device look-up."""

  def __init__(self, value_mapping, dtype=None, permute=None):
    from pycolab_b200 import observers
    self._value_mapping = value_mapping
    self._table, self._valid, self._is_3d = observers.value_table(value_mapping, dtype)
    try:
      self._permute = observers.check_permute(permute, self._is_3d, 'ObservationToArray')
    except ValueError:
      kind = ('1-D vectors' if self._is_3d else 'scalars')
      nums = ('0, 1, and 2' if self._is_3d else '0 and 1')
      raise ValueError(
          'When the value mapping contains {}, the permute argument to the '
          'ObservationToArray constructor must be a list or tuple containing some '
          'permutation of the integers {}.'.format(kind, nums))

  def __call__(self, observation):
    out, unknown = _on_device(observation.board, self._table, self._valid, self._is_3d,
                              self._permute, want_unknown=True)
    if unknown:
      raise RuntimeError(
          'This ObservationToArray only knows array values for the characters {}, but it '
          'received an observation with a character not in that set'.format(
              str(''.join(self._value_mapping.keys()))))
    return out


class ObservationCharacterRepainter(object):
  """Repaint characters through a mapping (rendering.py:304-406): returns an
  `Observation` whose layers follow the repainted board."""

  def __init__(self, character_mapping):
    from pycolab_b200 import observers
    self._character_mapping = character_mapping
    self._table = observers.repaint_table(character_mapping)

  def __call__(self, original_observation):
    # Upstream repaints through an ObservationToArray of the 128 ASCII codes, so a
    # byte >= 128 raises there.
    board, unknown = _on_device(original_observation.board, self._table, None, False, None,
                                want_unknown=True)
    if unknown:
      raise RuntimeError(
          'This ObservationCharacterRepainter only repaints ASCII characters, but it '
          'received an observation with a byte outside that set')
    chars = (set(original_observation.layers) - set(self._character_mapping)).union(
        self._character_mapping.values())
    return Observation(board=board, layers=LazyLayers(board, chars))


class ObservationToFeatureArray(object):
  """One-hot float32 feature planes for the chosen layers (rendering.py:545-661)."""

  def __init__(self, layers, permute=None):
    from pycolab_b200 import observers
    self._layers = layers
    self._permute = observers.check_permute(permute, True, 'ObservationToFeatureArray')

  def __call__(self, observation):
    if not any(l in observation.layers for l in self._layers):
      raise RuntimeError(
          'The layers argument to this ObservationToFeatureArray, {!r}, has no entry that '
          'refers to an actual feature in the input observation. Actual features in the '
          'observation are {!r}.'.format(self._layers, ''.join(sorted(observation.layers))))
    from pycolab_b200 import observers
    layers = observation.layers
    if (isinstance(layers, LazyLayers) and layers.board is observation.board and
        all(ord(c) < 128 for c in self._layers if c in layers)):
      # Occluded layers are `board == ord(c)`: one look-up per cell on the device.
      table = observers.feature_table(self._layers, present=layers)
      out, _ = _on_device(observation.board, table, None, True, self._permute)
      return out
    # Any other layers (un-occluded ones, or a user's dict) are copied as upstream
    # does, with zeros for layers the observation lacks.
    out = np.zeros((len(self._layers),) + observation.board.shape, dtype=np.float32)
    for index, character in enumerate(self._layers):
      if character in layers:
        np.copyto(out[index], layers[character])
    return out if self._permute is None else np.transpose(out, self._permute)


class BaseUnoccludedObservationRenderer(BaseObservationRenderer):
  """Same canvas protocol; layers ignore occlusion (rendering.py:187-301).  The
  board is still flattened on the GPU; the layers are the painted masks."""

  def render(self):
    board = render_on_device(self._backdrop, self._painted)
    layers = {}
    for ch in self._chars:
      mask = self._backdrop == ord(ch)
      for kind, painted_ch, data in self._painted:
        if painted_ch != ch:
          continue
        if kind == 'drape':
          mask = mask | data
        else:
          mask = mask.copy()
          mask[data] = True
      layers[ch] = mask
    return Observation(board=board, layers=layers)


def _launches(painted):
  """Split `painted` into runs, in order, that fit one pcl_render launch each."""
  from pycolab_b200 import _lib
  runs, sprites, drapes = [[]], 0, 0
  for item in painted:
    s, d = item[0] == 'sprite', item[0] == 'drape'
    if sprites + s > _lib.MAX_SPRITES or drapes + d > _lib.MAX_DRAPES:
      runs.append([])
      sprites = drapes = 0
    runs[-1].append(item)
    sprites, drapes = sprites + s, drapes + d
  return runs


def render_on_device(backdrop, painted, device=0):
  """`pcl_render` launches for a single canvas; returns uint8 [rows, cols].

  painted: [(kind, char, data)] in z-order, kind 'sprite' (data = (row, col)) or
  'drape' (data = bool mask).  A character painted several times occupies
  several z slots upstream; here each paint call gets its own slot too.  More
  paint calls than one launch holds are rendered in successive launches, each
  painting over the board the previous one made.
  """
  rows, cols = backdrop.shape
  # Each paint call gets a private slot code so repeated characters keep their
  # own z rank; the real character is restored after the launch.  The codes are
  # bytes that neither the backdrop nor any painted character uses, so the
  # restore touches painted cells only.
  used = set(np.unique(backdrop).tolist()) | set(ord(ch) for _, ch, _ in painted)
  free = [v for v in list(range(128, 256)) + list(range(128)) if v not in used]
  runs = _launches(painted)
  need = max(len(run) for run in runs)
  if need > len(free):
    raise ValueError('{} paint calls in one launch need {} free byte values for their '
                     'z slots; the backdrop and the painted characters leave {}'.format(
                         need, need, len(free)))
  board = np.array(backdrop, dtype=np.uint8)
  for run in runs:
    board = _render_once(board, run, free[:len(run)], device)
  return board


def _render_once(backdrop, painted, slots, device):
  """One `pcl_render` launch painting `painted` over `backdrop` with z slot codes
  `slots` (one per paint call)."""
  import torch
  from pycolab_b200 import _lib
  lib = _lib.load()
  rows, cols = backdrop.shape
  pitch = (cols + 15) // 16 * 16
  sprites = [(c, d) for k, c, d in painted if k == 'sprite']
  drapes = [(c, d) for k, c, d in painted if k == 'drape']
  spec = _lib.Spec()
  spec.abi_version, spec.program = _lib.ABI_VERSION, _lib.PROG_NONE
  spec.rows, spec.cols, spec.pitch = rows, cols, pitch
  spec.n_sprites, spec.n_drapes = len(sprites), len(drapes)
  sprite_i = drape_i = 0
  real = np.arange(256, dtype=np.uint8)
  for (kind, ch, _), slot in zip(painted, slots):
    real[slot] = ord(ch)
    if kind == 'sprite':
      spec.sprite_char[sprite_i] = slot
      sprite_i += 1
    else:
      spec.drape_char[drape_i] = slot
      drape_i += 1
  dev = torch.device('cuda', device)
  handle = C.c_void_p()
  _lib.check(lib.pcl_create(C.byref(spec), 1, device, C.byref(handle)), 'pcl_create')
  try:
    bd = np.zeros((1, rows, pitch), dtype=np.uint8)
    bd[0, :, :cols] = backdrop
    cur = np.zeros((1, max(1, len(drapes)), rows, pitch), dtype=np.uint8)
    for i, (_, mask) in enumerate(drapes):
      cur[0, i, :, :cols] = mask
    rec = np.zeros((1, max(1, len(sprites)), _lib.SPRITE_WORDS), dtype=np.int32)
    for i, (_, (r, c)) in enumerate(sprites):
      rec[0, i, _lib.S_ROW], rec[0, i, _lib.S_COL], rec[0, i, _lib.S_FLAGS] = r, c, 1
    t_bd = torch.from_numpy(bd).to(dev)
    t_cur = torch.from_numpy(cur).to(dev)
    t_rec = torch.from_numpy(rec).to(dev)
    t_z = torch.tensor([list(slots) or [0]], dtype=torch.uint8, device=dev)
    t_out = torch.zeros((1, rows, pitch), dtype=torch.uint8, device=dev)
    stream = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    _lib.check(lib.pcl_render(handle, t_bd.data_ptr(), 0, t_cur.data_ptr(),
                              t_rec.data_ptr(), t_z.data_ptr(), t_out.data_ptr(), stream),
               'pcl_render')
    torch.cuda.synchronize(dev)
    board = t_out[0, :, :cols].cpu().numpy()
  finally:
    lib.pcl_destroy(handle)
  return real[board]
