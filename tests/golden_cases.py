"""Load golden fixtures (tests/golden/*.npz) and rebuild their environments."""

import glob
import json
import os

import numpy as np

import trajectory as tj
from oracle import games

GOLDEN_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')


def names(prefix):
  return sorted(os.path.basename(p)[:-4]
                for p in glob.glob(os.path.join(GOLDEN_DIR, prefix + '*.npz')))


def load(name):
  with np.load(os.path.join(GOLDEN_DIR, name + '.npz')) as z:
    return {k: z[k] for k in z.files}


def config_of(g):
  return json.loads(bytes(g['config']).decode())


def scrolly_art(g):
  return (tj.u8_to_art(g['maze_art']), tj.u8_to_art(g['board_art']),
          chr(int(g['beneath'][0])))


def warehouse_art(g):
  wlb = g['what_lies_beneath']
  wlb = chr(int(wlb[0, 0])) if wlb.shape == (1, 1) else tj.u8_to_art(wlb)
  return tj.u8_to_art(g['art']), wlb


def fixture_kwargs(g):
  """kwargs for oracle.games.make_fixture_world / the facade equivalent."""
  cfg = config_of(g)
  scrollys = {}
  for ch, kw in cfg['scrollys'].items():
    key = {'#': 'pattern_hash', '@': 'pattern_at'}[ch]
    scrollys[ch] = dict(pattern=g[key].astype(bool),
                        corner=tuple(kw['corner']),
                        margins=None if kw['margins'] is None
                        else tuple(kw['margins']))
    if 'group' in kw:                    # named scrolling group (fixture_groups_*)
      scrollys[ch]['group'] = kw['group']
  return dict(art=tj.u8_to_art(g['art']),
              what_lies_beneath=cfg['what_lies_beneath'],
              walkers=cfg['walkers'], scrollys=scrollys, drapes=cfg['drapes'],
              update_schedule=cfg['schedule'], z_order=cfg['z_order']), cfg


def new_directive_row(row, n):
  """A stored action row of the `fixture_directives_*` goldens (n motions, reward
  or INT32_MIN, terminate 0/1, z_move_this or -1, z_in_front_of or 0) in the
  device's current layout: n motions + (opcode, argument) directive pairs
  (include/pcl.h PCL_DIR_*), same call order: reward, terminate, z-order."""
  from pycolab_b200 import _lib
  row = [int(x) for x in row]
  out, dirs = row[:n], []
  reward, term, z_this, z_that = row[n:n + 4]
  if reward != -(2 ** 31):
    dirs += [_lib.DIR_ADD_REWARD, reward]
  if term:
    dirs += [_lib.DIR_TERMINATE, 0]      # f32 bits of 0.0
  if z_this >= 0:
    dirs += [_lib.DIR_Z_ORDER, z_this | (z_that << 8)]
  dirs += [0] * (2 * _lib.FIXTURE_DIRECTIVES - len(dirs))
  return out + dirs
