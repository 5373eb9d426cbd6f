#!/usr/bin/env python
"""L2-resident and DRAM bandwidth of this H100, for setting a kernel's traffic against.

Two probes of tools/probes/l2_copy.cu, 16-byte accesses, loads through L2 only:
  * copy: ping-pong between two equal buffers; counted bytes = bytes read + bytes written;
  * read: a read-only sweep of one buffer (the step kernels' traffic is mostly reads).
At footprints well inside the 50 MB L2 (both copy buffers together), each launch makes
enough passes over the buffer to take tens of microseconds, so launch gaps are a small
share of the time; the DRAM point uses buffers of 1 GiB each and one pass per launch.
K launches are captured in one CUDA graph and timed with one CUDA event pair; the
number is the median of 5 graph replays after a warm-up replay.

The CUDA source is compiled with nvcc into a temporary directory at run time.

    python tools/l2_probe.py [--out profiles/h100_l2_probe.json]
"""
import argparse
import ctypes
import json
import os
import shutil
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

MB = 1 << 20
L2_FOOTPRINTS_MB = (4, 8, 16, 24)        # bytes of both copy buffers together / read buffer
DRAM_BUFFER = 1 << 30                    # per buffer
L2_BYTES_PER_LAUNCH = 512 * MB           # bytes moved per launch at the L2 footprints


def build_probe(tmp):
  nvcc = os.path.join(os.environ.get('CUDA_HOME', '/usr/local/cuda'), 'bin', 'nvcc')
  if not os.path.exists(nvcc):
    nvcc = shutil.which('nvcc') or nvcc
  so = os.path.join(tmp, 'l2_copy.so')
  subprocess.check_call([nvcc, '-gencode', 'arch=compute_90a,code=sm_90a', '-O3', '-shared',
                         '-Xcompiler', '-fPIC', '-cudart', 'static', '-o', so,
                         os.path.join(ROOT, 'tools', 'probes', 'l2_copy.cu')])
  lib = ctypes.CDLL(so)
  lib.l2_ping_pong.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int64, ctypes.c_int,
                               ctypes.c_int, ctypes.c_void_p]
  lib.l2_read_sweep.argtypes = [ctypes.c_void_p, ctypes.c_int64, ctypes.c_int, ctypes.c_int,
                                ctypes.c_void_p, ctypes.c_void_p]
  return lib


def time_graph(torch, launch, K):
  """Median ms of one replay of a graph of K `launch()` calls."""
  s = torch.cuda.Stream()
  with torch.cuda.stream(s):
    launch()                                   # warm-up outside the capture
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
      for _ in range(K):
        launch()
  g.replay()
  torch.cuda.synchronize()
  ms = []
  for _ in range(5):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    g.replay()
    b.record()
    b.synchronize()
    ms.append(a.elapsed_time(b))
  return sorted(ms)[2]


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--launches', type=int, default=20, help='launches per graph (K)')
  ap.add_argument('--out', default=None, help='also write the JSON result to this file')
  args = ap.parse_args()
  import torch
  import bench
  from step_sweep import card
  if not torch.cuda.is_available():
    raise SystemExit('l2_probe needs a CUDA device')
  dev = torch.device('cuda', 0)
  torch.cuda.set_device(dev)
  sms = torch.cuda.get_device_properties(dev).multi_processor_count
  blocks = sms * 8                             # 2048 threads per SM
  tmp = tempfile.mkdtemp(prefix='l2_probe_')
  try:
    lib = build_probe(tmp)
    sink = torch.zeros(4, dtype=torch.uint8, device=dev)

    def stream():
      return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)

    def check(rc):
      if rc != 0:
        raise RuntimeError('probe launch failed: cudaError %d' % rc)

    def copy_tbs(half_bytes, passes):
      a = torch.ones(half_bytes, dtype=torch.uint8, device=dev)
      b = torch.zeros_like(a)
      n16 = half_bytes // 16
      ms = time_graph(torch, lambda: check(lib.l2_ping_pong(a.data_ptr(), b.data_ptr(), n16,
                                                            passes, blocks, stream())),
                      args.launches)
      return 2 * half_bytes * passes * args.launches / (ms * 1e-3) / 1e12

    def read_tbs(nbytes, passes):
      a = torch.ones(nbytes, dtype=torch.uint8, device=dev)
      ms = time_graph(torch, lambda: check(lib.l2_read_sweep(a.data_ptr(), nbytes // 16, passes,
                                                             blocks, sink.data_ptr(), stream())),
                      args.launches)
      return nbytes * passes * args.launches / (ms * 1e-3) / 1e12

    sampler = bench.ClockSampler(0)
    sampler.start()
    copy_tbs(8 * MB, 64)                       # bring the clocks up
    sampler.mark_begin()
    l2_copy, l2_read = {}, {}
    for f in L2_FOOTPRINTS_MB:
      l2_copy[f] = round(copy_tbs(f * MB // 2, L2_BYTES_PER_LAUNCH // (f * MB)), 3)
      l2_read[f] = round(read_tbs(f * MB, L2_BYTES_PER_LAUNCH // (f * MB)), 3)
    dram_copy = round(copy_tbs(DRAM_BUFFER, 1), 3)
    dram_read = round(read_tbs(DRAM_BUFFER, 1), 3)
    sampler.mark_end()
    clocks = sampler.stop()
  finally:
    shutil.rmtree(tmp, ignore_errors=True)
  out = dict(card(0), sm_count=sms, sm_mhz_loaded=clocks.get('sm_mhz'), blocks=blocks,
             threads_per_block=256, launches_per_graph=args.launches,
             l2_copy_tb_s={'%d_MB' % f: v for f, v in l2_copy.items()},
             l2_read_tb_s={'%d_MB' % f: v for f, v in l2_read.items()},
             l2_copy_tb_s_max=max(l2_copy.values()), l2_read_tb_s_max=max(l2_read.values()),
             dram_copy_tb_s=dram_copy, dram_read_tb_s=dram_read,
             dram_buffer_bytes=DRAM_BUFFER)
  line = json.dumps(out)
  print(line)
  if args.out:
    with open(args.out, 'w') as f:
      f.write(line + '\n')


if __name__ == '__main__':
  main()
