"""Generate the cropped post-processor goldens (tests/golden/windowobs_*.npz) from the
REAL reference.

Run where the reference pycolab is installed:

    python tests/golden/make_crop_observe_golden.py

Each file is one case of tests/crop_cases.py, cut to a few envs and frames: what
make_crop_golden.py records (inputs, and per cropper the reference's cropped board,
corner and layers each frame), and per cropper and processor of
tests/crop_observe_cases.py, what the reference's own ObservationToFeatureArray /
ObservationToArray / ObservationCharacterRepainter returned on those cropped
Observations, zeros where it raised RuntimeError, and which calls raised.
"""

import os
import sys

import numpy as np

from make_golden import save

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import crop_cases as cc            # noqa: E402
import crop_observe_cases as coc   # noqa: E402
import refdriver                   # noqa: E402


def main():
  cropping = refdriver._import()['cropping']
  from pycolab import rendering
  for name, B, T in coc.GOLDEN_CASES:
    c = dict(cc.BY_NAME[name], B=B, T=T)
    seq = cc.frames(c)
    per_cropper = [cc.reference(cropping, c, k, seq, range(B)) for k in c['croppers']]
    outputs = {}
    for k, frames_k in enumerate(per_cropper):
      for proc in coc.PROCESSORS:
        got = [[coc.reference_apply(rendering, proc, crops[e], lays[e]) for e in range(B)]
               for crops, _, lays in frames_k]
        # the shape and dtype of one env's output, where every call raised too
        like = coc.oracle_apply(proc, frames_k[0][0], frames_k[0][2])[0][0]
        arr = np.stack([np.stack([np.zeros_like(like) if g is None else g for g in row])
                        for row in got])
        raised = np.array([[g is None for g in row] for row in got])
        outputs[(k, proc['name'])] = (arr, raised)
    save(coc.GOLDEN_PREFIX + name, **coc.golden_arrays(c, seq, per_cropper, outputs))


if __name__ == '__main__':
  main()
