#!/usr/bin/env python
"""Throughput of the other BASELINE.json configurations on one GPU.

    python tools/bench_configs.py [warehouse80|marauders|scrolly64crop] ...

bench.py measures the headline configuration (configs[1]); this script times
the remaining ones the same way (R independent batches stepped round-robin so
the working set exceeds L2 where the state is large enough, K back-to-back steps
between one CUDA event pair) and prints one JSON line per configuration.
Results are copied into profiles/ by hand.
"""

import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def build(name):
  from pycolab_b200 import levels, lowering
  if name == 'warehouse80':
    from pycolab_b200.games import warehouse_manager as g
    games = [lowering.lower(g.make_game(levels.warehouse_level(100 + i))) for i in range(16)]
    return dict(games=games, batch=8192, n_actions=4, rotation=3,
                a_step=80 * 80 * 3 + 64 * 11 + 64, kernel='warehouse_step',
                what='warehouse_manager 80x80, 10 boxes, generated levels (configs[2])')
  if name == 'marauders':
    from pycolab_b200.games import extraterrestrial_marauders as g
    games = [lowering.lower(g.make_game(levels.marauders_level()))]
    return dict(games=games, batch=4096, n_actions=4, rotation=2,
                a_step=16 * 39 * 6 + 64 * 7 + 64, kernel='marauders_step',
                what='extraterrestrial_marauders stock 16x39, 4096 envs per GPU (configs[3] '
                     '= 16384 over 4 GPUs)')
  if name == 'scrolly64crop':
    from pycolab_b200.games import scrolly_maze as g
    games = [lowering.lower(g.make_game(*levels.scrolly_maze_level(1000 + i)))
             for i in range(32)]
    return dict(games=games, batch=8192, n_actions=5, rotation=3,
                a_step=64 * 64 * 6 + 64 * 4 + 64 + 81, kernel='scrolly_maze_step + crop_kernel',
                crop=True,
                what='scrolly_maze 64x64 + ScrollingCropper 9x9 egocentric, 8192 envs per GPU '
                     '(configs[4] = 65536 over 8 GPUs)')
  if name == 't_maze':
    from pycolab_b200.games import t_maze as g
    games = []
    for i in range(6):                    # six generated worlds, level 4, 100-frame episodes
      maze, cue = levels.t_maze_level(i)
      games.append(lowering.lower(g.make_game(4, False, 100, 5, 10, maze_art=maze,
                                              cue_art=cue)))
    return dict(games=games, batch=4096, actions=[1, 2, 3, 4, 5], rotation=3,
                a_step=7 * 16 + 4 * (8 + 6 * 8 + 16) + 7 * 2 * 4 + 14,
                kernel='t_maze_step', float_reward=True,
                what='research/lp-rnn/t_maze level 4, six generated 77x191 worlds, 7x11 board, '
                     '4096 envs, timeout 100 frames: every env redraws its cue and 191x77 '
                     'speckle once per 101 steps')
  raise SystemExit('unknown config %r' % name)


def run(name, steps=600, warmup=30):
  import torch
  from pycolab_b200 import batched
  cfg = build(name)
  dev = torch.device('cuda', 0)
  B, R = cfg['batch'], cfg['rotation']
  engines = [batched.BatchedEngine(cfg['games'], batch=B, device=0, env_offset=r * B,
                                   rng_seed=7) for r in range(R)]
  for e in engines:
    e.its_showtime()
  crop_spec = None
  if cfg.get('crop'):
    crop_spec = batched.scrolling_crop_spec(9, 9, 0, pad_char=' ',
                                            scroll_margins=(None, None))
  rs = np.random.RandomState(1)
  if 'actions' in cfg:
    acts_np = rs.choice(cfg['actions'], size=(warmup + steps, B)).astype(np.int32)
  else:
    acts_np = rs.randint(0, cfg['n_actions'], size=(warmup + steps, B)).astype(np.int32)
  acts = torch.from_numpy(acts_np).to(dev)

  def step(t, i):
    eng = engines[i % R]
    eng.play(acts[t])
    if crop_spec is not None:
      eng.crop(crop_spec)

  for t in range(warmup):
    step(t, t)
  torch.cuda.synchronize()
  a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  l0 = sum(e.launch_count() for e in engines)
  a.record()
  for t in range(steps):
    step(warmup + t, t)
  b.record()
  torch.cuda.synchronize()
  ms = a.elapsed_time(b) / steps
  launches = sum(e.launch_count() for e in engines) - l0
  if cfg.get('float_reward'):
    # the host-buffer entry points carry an int32 reward and refuse this program: no e2e
    # leg; instead the cost of the restart draws, a pcl_reset of every env (cue + speckle)
    n_reset = 20
    torch.cuda.synchronize()
    a.record()
    for _ in range(n_reset):
      engines[0].reset()
    b.record()
    torch.cuda.synchronize()
    reset_ms = a.elapsed_time(b) / n_reset
    print(json.dumps({
        'config': name, 'workload': cfg['what'], 'batch': B, 'rotation': R,
        'metric': 'env_steps_per_sec', 'value': B / (ms / 1000.0), 'ms_per_step': ms,
        'steps': steps, 'gpu_launches': launches, 'reset_all_ms': reset_ms,
        'env_errors': max(int(e.error_codes().abs().max()) for e in engines)}))
    return

  # End to end: pinned host actions in, (board or crop) + scalars out.
  eng = engines[0]
  pin = lambda shape, dt: torch.zeros(shape, dtype=dt).pin_memory()
  h_act = pin((B,), torch.int32)
  d_act = torch.zeros((B,), dtype=torch.int32, device=dev)
  h_crop = pin((B, 9, 9), torch.uint8)
  h_rew, h_done = pin((B,), torch.int32), pin((B,), torch.uint8)
  n_e2e = 100
  torch.cuda.synchronize()
  t0 = time.perf_counter()
  for t in range(n_e2e):
    e = engines[t % R]
    if crop_spec is None:
      e.play_host(acts_np[warmup + t])
    else:
      h_act.numpy()[:] = acts_np[warmup + t]
      d_act.copy_(h_act, non_blocking=True)
      res = e.play(d_act)
      h_crop.copy_(e.crop(crop_spec), non_blocking=True)
      h_rew.copy_(res.reward, non_blocking=True)
      h_done.copy_(res.done, non_blocking=True)
      torch.cuda.synchronize()
  e2e_s = time.perf_counter() - t0
  peaks = {}
  try:
    peaks = json.load(open(os.path.join(ROOT, 'MEASURED_PEAKS.json')))
  except (OSError, ValueError):
    pass
  peak = float(peaks.get('hbm_gbs', 3350.0))         # H100 SXM data sheet HBM3
  achieved = B * cfg['a_step'] / (ms / 1000.0) / 1e9
  out_bytes = B * (81 + 5) if crop_spec is not None else B * (eng.rows * eng.pitch + 10)
  print(json.dumps({
      'config': name, 'workload': cfg['what'], 'batch': B, 'rotation': R,
      'metric': 'env_steps_per_sec', 'value': B / (ms / 1000.0), 'ms_per_step': ms,
      'steps': steps, 'gpu_launches': launches,
      'e2e': {'value': B * n_e2e / e2e_s, 'h2d_bytes_per_step': B * 4,
              'd2h_bytes_per_step': out_bytes},
      'roofline': {'kernel': cfg['kernel'], 'bound': 'hbm', 'achieved': achieved,
                   'peak': peak, 'unit': 'GB/s', 'frac': achieved / peak,
                   'algorithmic_bytes_per_launch': B * cfg['a_step']},
      'env_errors': max(int(e.error_codes().abs().max()) for e in engines)}))


if __name__ == '__main__':
  for name in (sys.argv[1:] or ['warehouse80', 'marauders', 'scrolly64crop']):
    run(name)
