"""Generate the cropper goldens (tests/golden/cropgrid_*.npz) from the REAL reference.

Run where the reference pycolab is installed:

    python tests/golden/make_crop_golden.py

Each file is one case of tests/crop_cases.py, cut to a few envs and frames: its inputs
(boards, sprite positions and visibility, drape curtains, episode counters) and, per
cropper, what the reference's own ScrollingCropper / FixedCropper returned each frame on
a duck-typed engine: the cropped board, the window corner and every cropped layer.
"""

import os
import sys

from make_golden import save

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import crop_cases as cc     # noqa: E402
import refdriver            # noqa: E402

# (case of crop_cases.CASES, envs, frames)
CASES = (('b8x14_w4x6', 3, 12), ('b5x7_w3x5_b4099', 3, 10), ('b37x1_w1x5_pad', 3, 10),
         ('b32x32_w5x7_plot', 2, 8), ('b8x14_fixed', 2, 6))


def main():
  cropping = refdriver._import()['cropping']
  for name, B, T in CASES:
    c = dict(cc.BY_NAME[name], B=B, T=T)
    seq = cc.frames(c)
    per_cropper = [cc.reference(cropping, c, k, seq, range(B)) for k in c['croppers']]
    save(cc.GOLDEN_PREFIX + name, **cc.golden_arrays(c, seq, per_cropper))


if __name__ == '__main__':
  main()
