"""What seeding generators costs: the constructor's host loop against the seeding kernel, and
reset(seeds=) on the device.

Workload: t_maze (two generator slots per env: Python's `random` for the cue, NumPy's for the
speckle) at 4096 and 65 536 envs.
  constructor: the host words of every env (`batched._mt_state` per env and slot, what the
    constructor computed before, and still computes for seeds outside [0, 2**32)) against
    `BatchedEngine(..., rng_seed=s)`, which seeds through pcl_seed_rng; host wall-clock time,
    the engine's ending in a device synchronise, best of `--repeats`.
  seed kernel: pcl_seed_rng alone over every env, CUDA events around `--launches` launches.
  seeded reset: the two launches reset(mask, seeds=) makes, pcl_seed_rng and pcl_reset, with
    half the envs selected and the seeds already a [B] device tensor (reset() also checks
    the seeds' range on the host, which a captured call skips), CUDA events around
    `--launches` of them; and the same reset without the seeding (pcl_reset alone), for
    comparison.
Prints JSON lines: first the card's name, power limit and maximum SM clock, read in the same
run; `--out` appends them to a file.

    python tools/seed_bench.py [--repeats 3] [--launches 200] [--out FILE]
"""

import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

import numpy as np                                              # noqa: E402

from compiled_bench import card                                # noqa: E402
from pycolab_b200 import batched, lowering                     # noqa: E402
from pycolab_b200.games import t_maze                          # noqa: E402

SIZES = (4096, 65536)


def events_us(fn, launches):
  import torch
  fn()
  torch.cuda.synchronize()
  a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  a.record()
  for _ in range(launches):
    fn()
  b.record()
  b.synchronize()
  return a.elapsed_time(b) * 1000.0 / launches


def main():
  import torch
  ap = argparse.ArgumentParser()
  ap.add_argument('--repeats', type=int, default=3)
  ap.add_argument('--launches', type=int, default=200)
  ap.add_argument('--out', default=None)
  args = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit('seed_bench measures on a CUDA device; none is available')
  lines = [dict(card=card())]
  game = lowering.lower(t_maze.make_game(1, False))
  streams = game.rng_streams
  for B in SIZES:
    host = []
    for _ in range(args.repeats):
      t0 = time.perf_counter()
      np.stack([np.concatenate([batched._mt_state(s, 7 + e) for s in streams])
                for e in range(B)])
      host.append(time.perf_counter() - t0)
    kernel, eng = [], None
    for _ in range(args.repeats):
      del eng
      torch.cuda.synchronize()
      t0 = time.perf_counter()
      eng = batched.BatchedEngine([game], batch=B, rng_seed=7)
      torch.cuda.synchronize()
      kernel.append(time.perf_counter() - t0)
    eng.its_showtime()
    seeds = torch.randint(0, 2 ** 32, (B,), dtype=torch.int64, device='cuda')
    d_seeds = eng._seed_tensor(seeds)
    mask = (torch.arange(B, device='cuda') % 2).to(torch.uint8)
    seed_us = events_us(lambda: eng._seed(None, d_seeds), args.launches)

    def seeded_reset():
      eng._seed(mask, d_seeds)
      eng.reset(mask)
    reset_us = events_us(seeded_reset, args.launches)
    plain_us = events_us(lambda: eng.reset(mask), args.launches)
    lines.append(dict(envs=B, slots=len(streams), streams=list(streams),
                      constructor_host_words_s=min(host), constructor_engine_s=min(kernel),
                      seed_kernel_us=seed_us, seeded_reset_half_masked_us=reset_us,
                      reset_half_masked_us=plain_us))
  for line in lines:
    print(json.dumps(line))
  if args.out:
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, 'a') as f:
      for line in lines:
        f.write(json.dumps(line) + '\n')


if __name__ == '__main__':
  main()
