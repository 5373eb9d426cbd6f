"""What keeping episode returns on the device costs on bench.py's C2 workload.

C2: scrolly_maze on bench.py's 32 generated 64x64 levels (129x129 worlds), 4096 envs in one
handle, actions drawn from 0..5 with a 1 % quit (so episodes end and restart throughout).
Two engines, one made with track_episodes=True and one without, alternated `--rounds`
times:
  play: `--steps` play()s captured as one CUDA graph, replayed `--repeats` times, one CUDA
    event pair around each replay (as bench.py times its graph): us per step.
  rollout: one T = `--T` rollout() captured as a CUDA graph (with episodes= on the
    tracking engine, which then also keeps [T, B] returns and lengths), replayed
    `--repeats` times: us per step.
Prints JSON lines: first the card's name, power limit and maximum SM clock, read in the same
run, and last the SM clock sampled right after the timings; `--out` appends them to a file.

    python tools/episode_bench.py [--steps 1000] [--T 128] [--repeats 5] [--rounds 2] [--out FILE]
"""

import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

import numpy as np                                              # noqa: E402

from compiled_bench import card                                # noqa: E402
from time_limit_bench import BATCH, N_LEVELS, c2_games         # noqa: E402
from pycolab_b200 import batched                               # noqa: E402


def sm_clock():
  out = subprocess.run(['nvidia-smi', '--query-gpu=clocks.sm', '--format=csv,noheader'],
                       capture_output=True, text=True)
  return out.stdout.strip().splitlines()[0] if out.returncode == 0 else 'unknown'


def replay_us(g, steps, repeats):
  import torch
  g.replay()
  torch.cuda.synchronize()
  out = []
  for _ in range(repeats):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    g.replay()
    b.record()
    b.synchronize()
    out.append(a.elapsed_time(b) * 1000.0 / steps)
  return out


def play_graph(eng, actions):
  import torch
  for t in range(actions.shape[0]):     # warm-up: every launch shape the graph holds
    eng.play(actions[t])
  torch.cuda.synchronize()
  g = torch.cuda.CUDAGraph()
  with torch.cuda.graph(g):
    for t in range(actions.shape[0]):
      eng.play(actions[t])
  return g


def rollout_graph(eng, actions):
  """(graph, buffers): a captured rollout and the Trajectory and Episodes it writes into.
  The graph holds their addresses but not the tensors: the caller keeps the buffers for as
  long as it replays the graph, or the replays write into whatever reuses that memory."""
  import torch
  ep = eng.new_episodes(actions.shape[0]) if eng.episode_return is not None else None
  traj = eng.rollout(actions, episodes=ep)
  torch.cuda.synchronize()
  g = torch.cuda.CUDAGraph()
  with torch.cuda.graph(g):
    eng.rollout(actions, out=traj, episodes=ep)
  return g, (traj, ep)


def main():
  import torch
  ap = argparse.ArgumentParser()
  ap.add_argument('--steps', type=int, default=1000)
  ap.add_argument('--T', type=int, default=128)
  ap.add_argument('--repeats', type=int, default=5)
  ap.add_argument('--rounds', type=int, default=2)
  ap.add_argument('--out', default=None, help='also append the lines to this file')
  args = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit('episode_bench needs a CUDA device: nothing is timed without one')
  lines = [{'card': card(), 'device': torch.cuda.get_device_name(0)}]
  print(json.dumps(lines[0]), flush=True)
  games = c2_games()
  rs = np.random.RandomState(1234)
  acts = rs.choice(6, size=(args.steps, BATCH), p=[.198] * 5 + [.01]).astype(np.int32)
  actions = torch.from_numpy(acts).cuda()
  workload = 'C2: scrolly_maze 64x64, %d levels, %d envs, one handle, 1%% quits' % (
      N_LEVELS, BATCH)
  engines = {}
  for track in (False, True):
    eng = batched.BatchedEngine(games, batch=BATCH, track_episodes=track)
    eng.its_showtime()
    g_roll, buffers = rollout_graph(eng, actions[:args.T])
    engines[track] = (eng, play_graph(eng, actions), g_roll, buffers)
  for r in range(args.rounds):
    for track in (False, True):
      eng, g_play, g_roll, _ = engines[track]
      play = replay_us(g_play, args.steps, args.repeats)
      roll = replay_us(g_roll, args.T, args.repeats)
      line = dict(workload=workload, round=r, track_episodes=track,
                  play_steps=args.steps, play_us_per_step=[round(x, 3) for x in play],
                  play_median_us=float(np.median(play)),
                  rollout_T=args.T, rollout_us_per_step=[round(x, 3) for x in roll],
                  rollout_median_us=float(np.median(roll)))
      print(json.dumps(line), flush=True)
      lines.append(line)
  lines.append({'sm_clock_after': sm_clock()})
  print(json.dumps(lines[-1]), flush=True)
  for eng, _, _, _ in engines.values():
    eng.close()
  if args.out:
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, 'a') as f:
      for line in lines:
        f.write(json.dumps(line) + '\n')


if __name__ == '__main__':
  main()
