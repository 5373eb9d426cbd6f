#!/usr/bin/env python
"""Launch-size sweep of the C2 scrolly_maze step: microseconds per step and nanoseconds
per env at batch sizes on both sides of the one-wave limit of `scrolly_maze_step`.

At 8 resident 4-warp blocks per SM, one wave on an H100's 132 SMs holds 4224 envs; at 7
it holds 3696.  A kernel whose time scales with the env count gives t(3696) close to
3696/4096 = 0.90 x t(4096); a launch that needs a tail wave shows a step instead:
t(3696) well below that and t(4096) close to t(4224).  4352 is one 128-env tail past
the 8-block wave.

Each size is timed like bench.py's headline: one CUDA graph of K step launches over 6
rotating batches (working set beyond the 50 MB L2), one event pair, median of 5
replays.  The library is the one `pycolab_b200._lib` loads (PCL_LIB_PATH selects
another build).

    python tools/step_sweep.py [--steps 1000] [--sizes 3696,4096,4224,4352,7392,8192]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card(index):
  q = subprocess.run(['nvidia-smi', '-i', str(index), '--query-gpu=name,power.limit,clocks.max.sm',
                      '--format=csv,noheader,nounits'], capture_output=True, text=True)
  name, limit, max_sm = [x.strip() for x in q.stdout.strip().split(',')]
  return {'gpu': name, 'power_limit_w': float(limit), 'sm_max_mhz': float(max_sm)}


def time_size(torch, dev, lowered, B, K, warm):
  import numpy as np
  import bench
  from pycolab_b200 import batched
  engines = [batched.BatchedEngine(lowered, batch=B, device=dev.index, env_offset=r * B)
             for r in range(bench.ROTATION)]
  for e in engines:
    e.its_showtime()
  acts = torch.from_numpy(np.random.RandomState(1234).randint(
      0, bench.ACTIONS, size=(warm + K, B)).astype(np.int32)).to(dev)
  timed = bench.Timed(torch, dev, lambda t: engines[t % bench.ROTATION].play(acts[t]), warm, K)
  if not timed.graphs:
    raise SystemExit('CUDA graph capture failed: ' + timed.path)
  sampler = bench.ClockSampler(dev.index)
  sampler.start()
  bench.ramp_clocks(torch, dev, timed, 0.3)
  timed.warm()
  sampler.mark_begin()
  ms = sorted(timed.time_ms(lambda: torch.cuda.synchronize(dev)) for _ in range(5))[2]
  sampler.mark_end()
  del timed, engines
  torch.cuda.synchronize(dev)
  return ms * 1e3 / K, sampler.stop()['sm_mhz']


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--steps', type=int, default=1000)
  ap.add_argument('--warmup', type=int, default=50)
  ap.add_argument('--sizes', default='3696,4096,4224,4352,7392,8192')
  args = ap.parse_args()
  import torch
  import bench
  from pycolab_b200 import _lib, lowering
  from pycolab_b200.games import scrolly_maze
  dev = torch.device('cuda', 0)
  torch.cuda.set_device(dev)
  lowered = [lowering.lower(scrolly_maze.make_game(*a)) for a in bench.make_levels(bench.N_LEVELS)]
  us, mhz = {}, {}
  for B in (int(s) for s in args.sizes.split(',')):
    us[B], mhz[B] = time_size(torch, dev, lowered, B, args.steps, args.warmup)
  out = dict(card(0), sm_mhz_loaded=mhz, lib=os.path.relpath(_lib.LIB_PATH, ROOT),
             steps=args.steps, rotation=bench.ROTATION,
             us_per_step={B: round(t, 3) for B, t in us.items()},
             ns_per_env={B: round(t * 1e3 / B, 3) for B, t in us.items()})
  if 3696 in us and 4096 in us:
    out['t3696_over_t4096'] = round(us[3696] / us[4096], 4)
    out['tail_gap_us'] = round(us[4096] - us[3696] * 4096 / 3696, 3)
  print(json.dumps(out))


if __name__ == '__main__':
  main()
