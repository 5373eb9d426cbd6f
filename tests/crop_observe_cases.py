"""Croppers feeding the observation post-processors, shared by the CPU and GPU tests.

`PROCESSORS` are upstream post-processor constructions (ObservationToFeatureArray over
occluded or un-occluded layers, ObservationToArray with scalar and vector mappings of
several dtypes and permutes, some missing a character, ObservationCharacterRepainter)
applied to the cropped observations of `crop_cases` frames.  `reference_apply` runs the
reference's own classes, `oracle_apply` the oracle's (`oracle.engine_model`) over a whole
batch of windows; the goldens (tests/golden/windowobs_*.npz) hold what the reference
returned, and which calls raised RuntimeError.
"""

import json
import os

import numpy as np

import crop_cases as cc

ALL = cc.BACKDROP + cc.SPRITES + cc.DRAPES


def _scalar(chars, f):
  return dict((ch, f(ch)) for ch in chars)


PROCESSORS = [
    dict(name='feat_occluded', kind='feature', layers='A.x#Q', permute=None, occluded=True),
    dict(name='feat_unoccluded_hwc', kind='feature', layers=' ByA.#x', permute=(1, 2, 0),
         occluded=False),
    dict(name='feat_unoccluded_wcr', kind='feature', layers='x.Ax', permute=(2, 0, 1),
         occluded=False),
    dict(name='arr_f32_scalar', kind='array', dtype='float32', permute=(1, 0),
         mapping=_scalar(ALL, lambda ch: ord(ch) / 4.0)),
    dict(name='arr_u8_vector', kind='array', dtype='uint8', permute=(2, 0, 1),
         mapping=_scalar(ALL, lambda ch: (ord(ch), 255 - ord(ch), ord(ch) % 7))),
    dict(name='arr_i64_no_hash', kind='array', dtype='int64', permute=None,
         mapping=_scalar(ALL.replace('#', ''), lambda ch: -ord(ch) * 3 ** 30)),
    dict(name='arr_f16_no_A', kind='array', dtype='float16', permute=(0, 2, 1),
         mapping=_scalar(ALL.replace('A', ''), lambda ch: (ord(ch) / 3.0, -ord(ch)))),
    dict(name='arr_bool', kind='array', dtype='bool', permute=None,
         mapping=_scalar(ALL, lambda ch: ch in '#x')),
    dict(name='repaint', kind='repaint', mapping={'.': 'x', 'A': '#', 'x': 'A'}),
]
BY_NAME = dict((p['name'], p) for p in PROCESSORS)

# (case of crop_cases.CASES, envs, frames): padded, fixed, off-board, two croppers; every
# case also runs the un-occluded processors on its cropped layers
GOLDEN_CASES = (('b8x14_w10x16_pad', 3, 6), ('b8x14_fixed', 2, 5), ('b31x33_w9x9_off', 3, 6),
                ('b32x32_two_croppers', 3, 6), ('b5x7_w3x5_b4099', 3, 6))
GOLDEN_PREFIX = 'windowobs_'


def reference_apply(rendering, proc, board, layers):
  """The reference's post-processor `proc` on one cropped Observation (board u8 [r, c],
  layers {char: bool [r, c]}: the cropper's layers, used as given by un-occluded feature
  processors; the others see the occluded layers of the board).  None if it raised
  RuntimeError."""
  if proc['kind'] == 'feature' and proc['occluded'] or proc['kind'] != 'feature':
    layers = dict((ch, board == ord(ch)) for ch in layers)
  obs = rendering.Observation(board=board, layers=layers)
  try:
    if proc['kind'] == 'feature':
      return rendering.ObservationToFeatureArray(proc['layers'], permute=proc['permute'])(obs)
    if proc['kind'] == 'array':
      return rendering.ObservationToArray(proc['mapping'], dtype=np.dtype(proc['dtype']),
                                          permute=proc['permute'])(obs)
    return rendering.ObservationCharacterRepainter(proc['mapping'])(obs).board
  except RuntimeError:
    return None


def _batch_permute(out, permute):
  return out if permute is None else np.transpose(out, [0] + [1 + i for i in permute])


def oracle_apply(proc, boards, layers=None):
  """The oracle's post-processor `proc` over a batch of windows (boards u8 [B, r, c];
  layers: per env {char: bool [r, c]}, the cropped un-occluded layers).  Returns (out
  [B, ...], raised): raised is True when the oracle raises RuntimeError for some env, and
  then out is that of the envs that do not raise, zeros for the others."""
  from oracle import engine_model as em
  if proc['kind'] == 'feature':
    obs_layers = None
    if not proc['occluded']:
      obs_layers = dict((ch, np.stack([lay[ch] for lay in layers])) for ch in layers[0])
    out = em.observation_to_feature_array(boards, proc['layers'], None, obs_layers)
    return _batch_permute(np.moveaxis(out, 0, 1), proc['permute']), False
  if proc['kind'] == 'repaint':
    return em.observation_repaint(boards, proc['mapping']), False
  known = np.zeros(256, bool)
  known[[ord(ch) for ch in proc['mapping']]] = True
  bad = ~known[boards].reshape(len(boards), -1).all(1)
  safe = np.where(bad[:, None, None], boards.dtype.type(ord(next(iter(proc['mapping'])))),
                  boards)
  out = em.observation_to_array(safe, proc['mapping'], np.dtype(proc['dtype']))
  out = out[None] if out.ndim == 3 else out                  # [depth, B, r, c]
  out = np.moveaxis(out, 0, 1)
  out[bad] = 0
  if not isinstance(next(iter(proc['mapping'].values())), tuple):
    out = out[:, 0]
  return _batch_permute(out, proc['permute']), bool(bad.any())


def golden_names():
  import glob
  return sorted(os.path.basename(p)[:-4]
                for p in glob.glob(os.path.join(cc.GOLDEN_DIR, GOLDEN_PREFIX + '*.npz')))


def golden_arrays(c, seq, per_cropper, outputs):
  """npz arrays: the crop_cases golden arrays of the case, and per cropper k and
  processor, the reference's outputs [T, B, ...] and raised flags [T, B]."""
  out = cc.golden_arrays(c, seq, per_cropper)
  out['processors'] = np.frombuffer(json.dumps([p['name'] for p in PROCESSORS]).encode(),
                                    np.uint8)
  for (k, name), (arr, raised) in outputs.items():
    out['out%d_%s' % (k, name)] = arr
    out['raised%d_%s' % (k, name)] = raised
  return out


def load_golden(name):
  """(case, frames, crops as crop_cases.load_golden, {(k, processor): (out, raised)})."""
  c, seq, want = cc.load_golden(name)
  with np.load(os.path.join(cc.GOLDEN_DIR, name + '.npz')) as z:
    names = json.loads(bytes(z['processors']).decode())
    outs = dict(((k, n), (z['out%d_%s' % (k, n)], z['raised%d_%s' % (k, n)]))
                for k in range(len(c['croppers'])) for n in names)
  return c, seq, want, outs
