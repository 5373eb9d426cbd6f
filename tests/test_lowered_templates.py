"""What `lowering.lower` makes for one level of every step program (tests/boundary_sweep.py),
field by field, against tests/golden/lowered_templates.json: spec bytes, template arrays, data
fields and which host hooks are set.  No GPU."""

import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, 'golden'))

import make_lowered_templates  # noqa: E402

GOLDEN = os.path.join(HERE, 'golden', 'lowered_templates.json')


def test_every_level_lowers_to_the_same_templates():
  with open(GOLDEN) as f:
    want = json.load(f)
  got = make_lowered_templates.digests()
  assert list(got) == list(want)
  differ = ['%s.%s' % (level, field) for level in want
            for field in sorted(set(want[level]) | set(got[level]))
            if want[level].get(field) != got[level].get(field)]
  assert not differ, 'lowered fields differ: ' + ', '.join(differ)
