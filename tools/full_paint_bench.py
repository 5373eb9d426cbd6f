#!/usr/bin/env python
"""The C2 step when every step is a full paint: bench.py's headline workload with each of
its 6 rotating batches writing two board buffers in turn.

`scrolly_maze_step` repaints only the changed cells when the board in the step's buffer
is the env's last render and neither window moves (scrolly_maze.cu, "Delta rendering").
With two buffers in turn no env ever finds its last render in the buffer it is given, so
every step takes the full path: this times that worst case beside the usual single
buffer.  Timing as bench.py's headline and tools/step_sweep.py: one CUDA graph of K
step launches, one event pair, median of 5 replays, rounds alternating the two modes.
The library is the one `pycolab_b200._lib` loads (PCL_LIB_PATH selects another build).

    python tools/full_paint_bench.py [--steps 1000] [--warmup 50] [--rounds 3]
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))


def time_mode(torch, dev, lowered, buffers, K, warm):
  import bench
  from pycolab_b200 import batched
  B = bench.BATCH_PER_GPU
  R = bench.ROTATION
  engines = [batched.BatchedEngine(lowered, batch=B, device=dev.index, env_offset=r * B)
             for r in range(R)]
  for e in engines:
    e.its_showtime()
  boards = [[e._board] + [torch.zeros_like(e._board) for _ in range(buffers - 1)] for e in engines]
  acts = torch.from_numpy(np.random.RandomState(1234).randint(
      0, bench.ACTIONS, size=(warm + K, B)).astype(np.int32)).to(dev)

  def step(t):
    e = engines[t % R]
    e._out.d_board = boards[t % R][(t // R) % buffers].data_ptr()
    e.play(acts[t])

  timed = bench.Timed(torch, dev, step, warm, K)
  if not timed.graphs:
    raise SystemExit('CUDA graph capture failed: ' + timed.path)
  bench.ramp_clocks(torch, dev, timed, 0.3)
  timed.warm()
  ms = sorted(timed.time_ms(lambda: torch.cuda.synchronize(dev)) for _ in range(5))[2]
  del timed, engines
  torch.cuda.synchronize(dev)
  return ms * 1e3 / K


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--steps', type=int, default=1000)
  ap.add_argument('--warmup', type=int, default=50)
  ap.add_argument('--rounds', type=int, default=3)
  args = ap.parse_args()
  import torch
  import bench
  from step_sweep import card
  from pycolab_b200 import _lib, lowering
  from pycolab_b200.games import scrolly_maze
  dev = torch.device('cuda', 0)
  torch.cuda.set_device(dev)
  lowered = [lowering.lower(scrolly_maze.make_game(*a)) for a in bench.make_levels(bench.N_LEVELS)]
  us = {'one_buffer': [], 'two_buffers': []}
  for _ in range(args.rounds):
    us['one_buffer'].append(round(time_mode(torch, dev, lowered, 1, args.steps, args.warmup), 3))
    us['two_buffers'].append(round(time_mode(torch, dev, lowered, 2, args.steps, args.warmup), 3))
  print(json.dumps(dict(card(0), lib=os.path.relpath(_lib.LIB_PATH, ROOT), steps=args.steps,
                        batch=bench.BATCH_PER_GPU, rotation=bench.ROTATION, us_per_step=us)))


if __name__ == '__main__':
  main()
