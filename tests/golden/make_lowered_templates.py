"""Write tests/golden/lowered_templates.json: per level of tests/boundary_sweep.py, one
digest per field of what `lowering.lower` makes (spec bytes, template arrays, data fields
and which host hooks are set), so a change to one program's host code names the field
it moved.  No GPU is needed.

Each level is lowered in a child process with PYTHONHASHSEED=0 (hello_world's update
order, and with it its sprite slots, follows set iteration) after seeding `random` and
`np.random` with 0 (apprehend and t_maze draw from them in their constructors).

  python tests/golden/make_lowered_templates.py
"""

import hashlib
import json
import os
import subprocess
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
OUT = os.path.join(HERE, 'lowered_templates.json')

ARRAYS = ('backdrop', 'sprites', 'drapes', 'plot', 'group_records')
ARRAY_DICTS = ('patterns', 'pattern_mutable', 'pattern_redraw', 'bits')
DATA = ('reward_type', 'float_reward', 'needs_rng', 'dynamic_z', 'backdrop_role',
        'scroll_groups', 'sprite_group', 'drape_group', 'actions_per_env', 'rng_streams')
HOOKS = ('curtain', 'layers', 'sync', 'action_row')


def _sha(*parts):
  h = hashlib.sha256()
  for p in parts:
    h.update(p if isinstance(p, bytes) else repr(p).encode('utf-8'))
  return h.hexdigest()[:16]


def _array(a):
  if a is None:
    return _sha(None)
  a = np.asarray(a)
  return _sha(a.dtype.str, a.shape, np.ascontiguousarray(a).tobytes())


def field_digests(game):
  """{field: digest} of one `LoweredGame`."""
  out = {'spec': _sha(bytes(game.make_spec(True)))}
  for name in ARRAYS:
    out[name] = _array(getattr(game, name))
  for name in ARRAY_DICTS:
    d = getattr(game, name)
    out[name] = _sha(*[x for k in sorted(d) for x in (k, _array(d[k]))])
  for name in DATA:
    value = getattr(game, name)
    out[name] = _sha(value.__name__ if isinstance(value, type) else value)
  out['hooks'] = _sha([h for h in HOOKS if getattr(game, h) is not None])
  return out


def _child():
  """Print {level: {field: digest}} for every level, as JSON."""
  import random
  import boundary_sweep
  from pycolab_b200 import lowering
  out = {}
  for name, make in boundary_sweep._games():
    random.seed(0)
    np.random.seed(0)
    out[name] = field_digests(lowering.lower(make()))
  print(json.dumps(out))


def digests():
  """{level: {field: digest}} from a child process with PYTHONHASHSEED=0."""
  env = dict(os.environ, PYTHONHASHSEED='0')
  text = subprocess.check_output([sys.executable, os.path.abspath(__file__), '--child'],
                                 env=env, cwd=ROOT)
  return json.loads(text.decode('utf-8').strip().splitlines()[-1])


def main():
  levels = digests()
  with open(OUT, 'w') as f:         # one line per level
    f.write('{\n' + ',\n'.join('%s: %s' % (json.dumps(level), json.dumps(fields, sort_keys=True))
                               for level, fields in levels.items()) + '\n}\n')
  print('%d levels -> %s' % (len(levels), OUT))


if __name__ == '__main__':
  for p in (ROOT, os.path.join(ROOT, 'tests')):
    if p not in sys.path:
      sys.path.insert(0, p)
  if sys.argv[1:] == ['--child']:
    _child()
  else:
    main()
