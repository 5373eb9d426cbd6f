"""Observation post-processors on the device (reference `pycolab/rendering.py:304-661`).

`ObservationCharacterRepainter`, `ObservationToArray` and
`ObservationToFeatureArray` are all "a function of the character, per cell", so
one kernel (`pcl_observe`, csrc/observe.cu) serves the three through a
[128, depth] table.  This module builds the tables from the reference's
constructor arguments and launches the kernel over a batch of boards; the
reference-named single-observation classes live in `rendering.py`.
"""

import ctypes as C

import numpy as np

from pycolab_b200 import _lib

# pcl_observe copies bits, so only an element's size picks the launch: the code of
# each size (include/pcl.h pcl_observe_spec.dtype), and the container it is moved in.
_CODE_OF_SIZE = {1: 0, 2: 5, 4: 1, 8: 3}
_CONTAINER = {1: np.uint8, 2: np.uint16, 4: np.uint32, 8: np.uint64}
MAX_PLANES = 32                  # planes one pcl_observe launch writes


def check_dtype(dtype):
  """`dtype` as a NumPy dtype if the device can produce it: bool, integers and
  floats of 1, 2, 4 or 8 bytes."""
  dt = np.dtype(dtype)
  if dt.kind not in 'biuf' or dt.itemsize not in _CODE_OF_SIZE:
    raise TypeError('ObservationToArray on the device supports bool, integer and float '
                    'outputs of 1, 2, 4 or 8 bytes, not {}'.format(dt))
  return dt


def value_table(value_mapping, dtype=None):
  """ObservationToArray's mapping (rendering.py:423-470) as (table [128, depth],
  valid u8 [128], is_3d).  Values are stored exactly as upstream stores them into
  its output array: masked assignment, one vector component at a time."""
  first = next(iter(value_mapping.values()))
  dt = check_dtype(dtype if dtype is not None else np.array(first).dtype)
  try:
    depth, is_3d = len(first), True
  except TypeError:
    depth, is_3d = 1, False
  planes = np.zeros((depth, 128), dtype=dt)
  valid = np.zeros((128,), dtype=np.uint8)
  for ch, value in value_mapping.items():
    code = ord(ch)
    if code > 127:
      raise ValueError('non-ASCII character {!r} in a value mapping'.format(ch))
    mask = np.arange(128) == code
    if is_3d:
      for layer, component in enumerate(value):
        planes[layer, mask] = component
    else:
      planes[:, mask] = value
    valid[code] = 1
  return np.ascontiguousarray(planes.T), valid, is_3d


def feature_table(layers, present=None):
  """ObservationToFeatureArray (rendering.py:545-661) over occluded layers
  (`board == ord(c)`): one-hot float32 planes.  A character outside `present` (the
  observation's layers; None = every character) or beyond ASCII gets a zero plane,
  as upstream fills layers the observation lacks with zeros."""
  table = np.zeros((128, len(layers)), dtype=np.float32)
  for d, ch in enumerate(layers):
    if ord(ch) < 128 and (present is None or ch in present):
      table[ord(ch), d] = 1.0
  return table


def repaint_table(character_mapping):
  """ObservationCharacterRepainter (rendering.py:304-357): identity LUT with the
  mapped characters replaced."""
  table = np.arange(128, dtype=np.uint8).reshape(128, 1).copy()
  for src, dst in character_mapping.items():
    table[ord(src), 0] = ord(dst)
  return table


def check_permute(permute, is_3d, who):
  if permute is None:
    return None
  permute = tuple(permute)
  want = [0, 1, 2] if is_3d else [0, 1]
  if sorted(permute) != want:
    raise ValueError(
        'The permute argument to the {} constructor must be a list or tuple containing '
        'some permutation of the integers {}.'.format(who, ', '.join(map(str, want))))
  return permute


def plane_chunks(depth):
  """[(first plane, planes)]: the pcl_observe launches of a `depth`-plane output."""
  return [(k0, min(MAX_PLANES, depth - k0)) for k0 in range(0, depth, MAX_PLANES)]


def _output(B, rows, cols, table, is_3d, permute, device):
  """(out, strides, t_table): the output tensor [B] + permuted([depth,] rows, cols) in
  the same-size unsigned container of `table.dtype`, the element strides of its
  unpermuted axes ({0: plane, 1: row, 2: column} for a 3-D output, {0: row, 1: column}
  otherwise) and the table on the device."""
  import torch
  depth = table.shape[1]
  size = table.dtype.itemsize
  base = [depth, rows, cols] if is_3d else [rows, cols]
  perm = list(permute) if permute is not None else list(range(len(base)))
  shape = [base[i] for i in perm]
  container = getattr(torch, np.dtype(_CONTAINER[size]).name)
  out = torch.empty([B] + shape, dtype=container, device=device)
  strides = list(out.stride())[1:]
  at = {base_dim: strides[perm.index(base_dim)] for base_dim in range(len(base))}
  t_table = torch.from_numpy(np.ascontiguousarray(table).view(_CONTAINER[size])).to(device)
  return out, at, t_table


def observe(lib, handle, board, rows, cols, table, valid, is_3d, permute, stream,
            unknown=None):
  """Run pcl_observe over `board` (u8 [B, rows, pitch] CUDA tensor).  Returns a
  CUDA tensor shaped [B] + permuted([depth,] rows, cols), in the same-size
  unsigned container of `table.dtype` (`torch_dtype` / `numpy_view` convert it).
  More than MAX_PLANES planes take one launch per MAX_PLANES."""
  import torch
  depth = table.shape[1]
  size = table.dtype.itemsize
  out, at, t_table = _output(board.shape[0], rows, cols, table, is_3d, permute, board.device)
  t_valid = None if valid is None else torch.from_numpy(valid).to(board.device)
  for k0, planes in plane_chunks(depth):
    spec = _lib.ObserveSpec(planes, _CODE_OF_SIZE[size], out.stride()[0],
                            at[0] if is_3d else 0,
                            at[1] if is_3d else at[0], at[2] if is_3d else at[1])
    chunk = t_table[:, k0:k0 + planes].contiguous()
    d_out = out.data_ptr() + (k0 * at[0] * size if is_3d else 0)
    _lib.check(lib.pcl_observe(handle, C.byref(spec), chunk.data_ptr(),
                               None if t_valid is None else t_valid.data_ptr(),
                               board.data_ptr(), d_out,
                               None if unknown is None else unknown.data_ptr(), stream),
               'pcl_observe')
  return out


def crop_observe(lib, handle, crop_spec, board, state, curtains, table, valid, is_3d, permute,
                 stream, unknown=None, planes=None, plane_of=None, pad_plane=-1, check=None):
  """Run pcl_crop_observe: crop_spec's window of `board` (u8 [B, rows, pitch] CUDA tensor),
  moved once as `pcl_crop_tracking` moves it (`state`: the cropper's corner array, None =
  the plot record's slot; `curtains`: the ctypes pointer array of tracked drapes' curtains,
  or None), through the [128, depth] `table` in one launch.  Returns what `observe`
  returns for a board of the window's shape.  With `planes` (u8 [B, n, rows, >= cols], one
  byte per column) the output planes are the un-occluded layers plane_of[d] (-1: zeros)
  of that window, off-board cells 1 in plane `pad_plane`.  `check(status, what)` judges
  the call's status (default `_lib.check`)."""
  import torch
  depth = table.shape[1]
  size = table.dtype.itemsize
  device = (board if planes is None else planes).device
  B = (board if planes is None else planes).shape[0]
  out, at, t_table = _output(B, crop_spec.rows, crop_spec.cols, table, is_3d, permute, device)
  t_valid = None if valid is None else torch.from_numpy(valid).to(device)
  spec = _lib.ObserveSpec(depth, _CODE_OF_SIZE[size], out.stride()[0], at[0] if is_3d else 0,
                          at[1] if is_3d else at[0], at[2] if is_3d else at[1])
  plane_args = (None, None, -1, 0, 0, 0)
  if planes is not None:
    assert planes.dtype == torch.uint8 and planes.stride()[3] == 1
    t_plane_of = torch.tensor(plane_of, dtype=torch.int32).to(device)
    plane_args = (planes.data_ptr(), t_plane_of.data_ptr(), int(pad_plane)) + tuple(
        planes.stride()[:3])
  status = lib.pcl_crop_observe(
      handle, C.byref(crop_spec), None if board is None else board.data_ptr(),
      None if state is None else state.data_ptr(), curtains, C.byref(spec),
      t_table.data_ptr(), None if t_valid is None else t_valid.data_ptr(), *plane_args,
      out.data_ptr(), None if unknown is None else unknown.data_ptr(), stream)
  if check is None:
    _lib.check(status, 'pcl_crop_observe', handle)
  else:
    check(status, 'pcl_crop_observe')
  return out


def torch_dtype(dtype):
  """The torch dtype of NumPy `dtype` (same size, same meaning)."""
  import torch
  dt = np.dtype(dtype)
  return torch.bool if dt == np.bool_ else getattr(torch, dt.name)


def numpy_view(out, dtype):
  """Host copy of an `observe` result as a NumPy array of `dtype`."""
  host = out.cpu().numpy()
  return host.view(dtype)
