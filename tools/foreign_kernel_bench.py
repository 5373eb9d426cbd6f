#!/usr/bin/env python
"""C2 steps that follow another kernel, so that none of them is chained to a step launch:
microseconds per (action-writing torch kernel + scrolly_maze step) pair.

  graph:  K pairs captured in one CUDA graph, a torch kernel writing each step's actions
          into one buffer just before the step (a policy's output in a training loop);
          one event pair, median of 5 replays.
  eager:  the same pairs launched one by one from the host, median of 5 rounds.

Each step keeps the full wait for the kernel before it.  The library is the one
`pycolab_b200._lib` loads (PCL_LIB_PATH selects another build).  Prints one JSON line.

    python tools/foreign_kernel_bench.py [--batch 4096] [--steps 1000] [--label NAME]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--batch', type=int, default=4096)
  ap.add_argument('--steps', type=int, default=1000)
  ap.add_argument('--label', default='', help='names the build in the output line')
  args = ap.parse_args()
  import numpy as np
  import torch
  import bench
  from pycolab_b200 import batched, lowering
  from pycolab_b200.games import scrolly_maze
  dev = torch.device('cuda', 0)
  B, K = args.batch, args.steps
  lowered = [lowering.lower(scrolly_maze.make_game(*a)) for a in bench.make_levels(bench.N_LEVELS)]
  eng = batched.BatchedEngine(lowered, batch=B, device=0)
  eng.its_showtime()
  acts = torch.from_numpy(np.random.RandomState(1234).randint(
      0, bench.ACTIONS, size=(K, B)).astype(np.int32)).to(dev)
  buf = torch.zeros(B, dtype=torch.int32, device=dev)

  def pairs():
    for t in range(K):
      torch.add(acts[t], 0, out=buf)
      eng.play(buf)

  def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize(dev)
    a.record()
    fn()
    b.record()
    torch.cuda.synchronize(dev)
    return a.elapsed_time(b) * 1e3 / K

  torch.cuda.synchronize(dev)
  g = torch.cuda.CUDAGraph()
  with torch.cuda.graph(g):
    pairs()
  sampler = bench.ClockSampler(0)
  sampler.start()
  for _ in range(3):
    g.replay()
  sampler.mark_begin()
  graph_us = sorted(timed(g.replay) for _ in range(5))[2]
  pairs()
  eager_us = sorted(timed(pairs) for _ in range(5))[2]
  sampler.mark_end()
  q = os.popen('nvidia-smi -i 0 --query-gpu=name,power.limit --format=csv,noheader,nounits').read()
  name, limit = [x.strip() for x in q.strip().split(',')]
  print(json.dumps({'gpu': name, 'power_limit_w': float(limit),
                    'sm_mhz': sampler.stop()['sm_mhz'], 'batch': B, 'steps': K,
                    'build': args.label,
                    'graph_us_per_pair': graph_us, 'eager_us_per_pair': eager_us}))


if __name__ == '__main__':
  main()
