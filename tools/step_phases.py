#!/usr/bin/env python
"""Where the time of one C2 scrolly_maze step goes, phase by phase, on the GPU.

Builds libpcl.so with -DPCL_STEP_STAMPS (the Makefile's flags otherwise) into a
temporary directory outside the tree.  In that build lane 0 of each warp of
`scrolly_maze_step` stores its SM's cycle counter at the phase boundaries below, and
%globaltimer at entry and exit (scrolly_maze.cu, PCL_STAMP).  Each size is timed like
bench.py's headline (tools/step_sweep.py: one CUDA graph of K step launches over 6
rotating batches); the stamps read afterwards are those of the graph's last launch,
one warp per env.  The production build (the in-tree library, or PCL_LIB_PATH) is
timed the same way, alternating with the stamp build, so the line shows whether the
stamps changed the step they describe.

Phases (cycles between consecutive stamps of one warp):
  prior_grid   entry -> griddepcontrol.wait returned (the previous launch of the stream)
  records      -> records in shared memory (first DRAM round trip)
  patch_bits   -> 5x5 wall / 3x3 coin patch bits loaded and shuffled (second round trip)
  groups       -> update groups 1 and 2 done
  copy_wait    -> backdrop tile and window copies landed (cp.async wait)
  seg_patch    -> records written back, segment words built, sprites patched
  paint        -> board stored
  cropper      -> cropper epilogue done (zero without a cropper)
A warp on the delta-rendering path stages nothing: its copy_wait is empty, seg_patch holds
the records write-back and the changed cells' stores, and paint is empty.

`paths` splits the warps by the path each took (PATHS below, one stamp word per warp):
their count, and the median and max of their work cycles (entry to end, less prior_grid)
and of their exit time, so the path whose warps end the launch shows.

    python tools/step_phases.py [--steps 1000] [--sizes 4096,128] [--rounds 2]
"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

PHASES = ('prior_grid', 'records', 'patch_bits', 'groups', 'copy_wait', 'seg_patch', 'paint',
          'cropper')
N_CLOCKS = len(PHASES) + 1          # slots 0..8: cycle stamps at the phase boundaries
T_IN, T_OUT, PATH, WORDS = 9, 10, 11, 12
# Values of the path slot (kPath* in scrolly_maze.cu).
PATHS = ('delta', 'delta_pickup', 'fell_back', 'full_paint', 'restart')


def build_stamps(out_dir):
  """The Makefile run on a copy of the sources, with the stamp switch added."""
  src = os.path.join(out_dir, 'pycolab_b200', 'csrc')
  shutil.copytree(os.path.join(ROOT, 'pycolab_b200', 'csrc'), src,
                  ignore=shutil.ignore_patterns('*.o', '*.so'))
  shutil.copytree(os.path.join(ROOT, 'include'), os.path.join(out_dir, 'include'))
  nvcc = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')
  res = subprocess.run(['make', '-C', src, '-j8', 'NVCC=%s -DPCL_STEP_STAMPS' % nvcc],
                       capture_output=True, text=True)
  if res.returncode != 0:
    raise SystemExit('stamp build failed:\n' + res.stderr[-4000:])
  return os.path.join(out_dir, 'pycolab_b200', 'libpcl.so')


def pct(x, q):
  import numpy as np
  return int(np.percentile(x, q)) if len(x) else None


def stamp_stats(raw):
  """Per-phase cycles and the warps' entry / exit spread from [n, WORDS] u32 stamps."""
  import numpy as np
  done = raw              # every env of the C2 workload steps (auto-reset: none is frozen)
  clk = done[:, :N_CLOCKS].astype(np.int64)
  d = (clk[:, 1:] - clk[:, :-1]) % (1 << 32)
  tot = (clk[:, -1] - clk[:, 0]) % (1 << 32)
  t0 = done[:, T_IN].astype(np.int64)
  ref = t0.min() if len(t0) else 0
  t_in = (t0 - ref) % (1 << 32)
  t_out = (done[:, T_OUT].astype(np.int64) - ref) % (1 << 32)
  work = tot - d[:, 0]
  paths = {}
  for k, name in enumerate(PATHS):
    sel = done[:, PATH] == k
    paths[name] = {'warps': int(sel.sum()),
                   'work_cycles': {'median': pct(work[sel], 50), 'max': pct(work[sel], 100)},
                   'exit_ns': {'median': pct(t_out[sel], 50), 'max': pct(t_out[sel], 100)}}
  return {
      'warps': int(len(done)),
      'cycles': {name: {'median': pct(d[:, i], 50), 'p90': pct(d[:, i], 90)}
                 for i, name in enumerate(PHASES)},
      'cycles_total': {'median': pct(tot, 50), 'p90': pct(tot, 90), 'max': pct(tot, 100)},
      'entry_ns': {'p10': pct(t_in, 10), 'p50': pct(t_in, 50), 'p90': pct(t_in, 90),
                   'max': pct(t_in, 100)},
      'exit_ns': {'min': pct(t_out, 0), 'p10': pct(t_out, 10), 'p50': pct(t_out, 50),
                  'p90': pct(t_out, 90), 'max': pct(t_out, 100)},
      'paths': paths,
  }


def worker(args):
  """Time each size with the library PCL_LIB_PATH names; read stamps if it has them."""
  import ctypes as C
  import numpy as np
  import torch
  import bench
  import step_sweep
  from pycolab_b200 import _lib, lowering
  from pycolab_b200.games import scrolly_maze
  dev = torch.device('cuda', 0)
  torch.cuda.set_device(dev)
  lib = _lib.load()
  read = getattr(lib, 'pcl_step_stamps', None)
  lowered = [lowering.lower(scrolly_maze.make_game(*a)) for a in bench.make_levels(bench.N_LEVELS)]
  out = {'us_per_step': {}, 'sm_mhz_loaded': {}, 'stamps': {}}
  for B in (int(s) for s in args.sizes.split(',')):
    us, mhz = step_sweep.time_size(torch, dev, lowered, B, args.steps, args.warmup)
    out['us_per_step'][B], out['sm_mhz_loaded'][B] = round(us, 3), mhz
    if read is not None:
      raw = np.zeros((B, WORDS), dtype=np.uint32)
      read.restype, read.argtypes = C.c_int, [C.c_void_p, C.c_int]
      if read(raw.ctypes.data, B) != 0:
        raise SystemExit('pcl_step_stamps failed')
      out['stamps'][B] = stamp_stats(raw)
  print(json.dumps(out))


def run_worker(lib_path, args):
  env = dict(os.environ)
  if lib_path:
    env['PCL_LIB_PATH'] = lib_path
  else:
    env.pop('PCL_LIB_PATH', None)
  cmd = [sys.executable, os.path.abspath(__file__), '--worker', '--sizes', args.sizes,
         '--steps', str(args.steps), '--warmup', str(args.warmup)]
  res = subprocess.run(cmd, env=env, check=True, capture_output=True, text=True)
  return json.loads(res.stdout.strip().splitlines()[-1])


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--steps', type=int, default=1000)
  ap.add_argument('--warmup', type=int, default=50)
  ap.add_argument('--sizes', default='4096,128')
  ap.add_argument('--rounds', type=int, default=2, help='production / stamp alternations')
  ap.add_argument('--worker', action='store_true', help=argparse.SUPPRESS)
  args = ap.parse_args()
  if args.worker:
    return worker(args)
  import step_sweep
  prod_lib = os.environ.get('PCL_LIB_PATH')
  with tempfile.TemporaryDirectory(prefix='pcl_stamps_') as tmp:
    stamp_lib = build_stamps(tmp)
    prod, stamped = [], []
    for _ in range(args.rounds):
      prod.append(run_worker(prod_lib, args))
      stamped.append(run_worker(stamp_lib, args))
  sizes = [int(s) for s in args.sizes.split(',')]
  us_prod = {B: sorted(r['us_per_step'][str(B)] for r in prod) for B in sizes}
  us_stamp = {B: sorted(r['us_per_step'][str(B)] for r in stamped) for B in sizes}
  out = dict(step_sweep.card(0), steps=args.steps, rounds=args.rounds,
             lib=os.path.relpath(prod_lib, ROOT) if prod_lib else 'pycolab_b200/libpcl.so',
             sm_mhz_loaded={B: sorted({r['sm_mhz_loaded'][str(B)] for r in prod + stamped})
                            for B in sizes},
             us_per_step_production=us_prod, us_per_step_stamps=us_stamp,
             stamp_overhead_pct={B: round(100.0 * (min(us_stamp[B]) / min(us_prod[B]) - 1), 2)
                                 for B in sizes},
             phases={B: stamped[-1]['stamps'][str(B)] for B in sizes})
  print(json.dumps(out))


if __name__ == '__main__':
  main()
