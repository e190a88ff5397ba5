#!/usr/bin/env python
"""A/B of engine knobs on ONE box: alternates the variants several times (fresh handle each) and prints medians.

    python tools/ab_bench.py BSB_BLOCK_THREADS=64 BSB_BLOCK_THREADS=128 [--track] [--host]
"""
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402
import bsuite_b200  # noqa: E402


def run(env_kv, track, host, steps=int(os.environ.get('AB_STEPS', '600'))):
  print('running', env_kv, flush=True)
  for k in [k for k in os.environ if k.startswith('BSB_')]:
    del os.environ[k]
  for kv in env_kv.split(','):
    k, v = kv.split('=')
    os.environ[k] = v
  env = bsuite_b200.load_from_id('deep_sea/11', batch=65536, device='cuda', seed=0, track_episodes=track)
  ring = [env.make_buffers() for _ in range(4)]
  if host:
    acts = torch.randint(0, 2, (64, 65536), dtype=torch.int32).pin_memory()
    hb = env.make_host_buffers()
    for i in range(20):
      env.step_host(acts[i % 64], hb, out=ring[i % 4])
    t0 = time.perf_counter()
    for i in range(steps // 3):
      env.step_host(acts[i % 64], hb, out=ring[i % 4])
    us = (time.perf_counter() - t0) / (steps // 3) * 1e6
  else:
    acts = torch.randint(0, 2, (64, 65536), device='cuda', dtype=torch.int32)
    for i in range(30):
      env.step(acts[i % 64], out=ring[i % 4])
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(steps):
      env.step(acts[i % 64], out=ring[i % 4])
    e1.record()
    torch.cuda.synchronize()
    us = e0.elapsed_time(e1) * 1e3 / steps
  env.close()
  return us


def main():
  variants = [a for a in sys.argv[1:] if '=' in a]
  track, host = '--track' in sys.argv, '--host' in sys.argv
  results = {v: [] for v in variants}
  for rep in range(5):
    for v in variants:
      results[v].append(run(v, track, host))
  for v in variants:
    r = results[v]
    print(f'{v:50s} median {statistics.median(r):7.2f} us  min {min(r):7.2f}  max {max(r):7.2f}  ({"host e2e" if host else "device"}; track={track})')


if __name__ == '__main__':
  main()
