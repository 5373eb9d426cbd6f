"""Write tests/golden/boundary_statuses.json: the C boundary's status for every case of
tests/boundary_sweep.py, one character per case (boundary_sweep.encode), from the library
`pycolab_b200._lib` loads (PCL_LIB_PATH picks another build).  No GPU is needed.

  python tests/golden/make_boundary_statuses.py
"""

import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
for p in (ROOT, os.path.join(ROOT, 'tests')):
  if p not in sys.path:
    sys.path.insert(0, p)

import boundary_sweep  # noqa: E402

OUT = os.path.join(HERE, 'boundary_statuses.json')


def main():
  statuses = boundary_sweep.sweep()
  levels = boundary_sweep.encode(statuses)
  with open(OUT, 'w') as f:         # one line per level
    f.write('{\n' + ',\n'.join('%s: %s' % (json.dumps(level), json.dumps(chars))
                               for level, chars in levels.items()) + '\n}\n')
  print('%d cases -> %s' % (len(statuses), OUT))


if __name__ == '__main__':
  main()
