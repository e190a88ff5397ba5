#!/usr/bin/env python
"""The full 468-id sweep as one handle per bsuite_id (`SweepBatch`, 468 handles) against one pack per experiment
(`SweepBatch(packed=True)`, 23 handles), on one GPU.

    python tools/bench_sweep_packed.py [--lanes 256 1024] [--steps 1 16] [--iters 20] [--rounds 5]

For each lanes-per-setting size and rollout length T: the time of one lock-step (every id advanced T steps), eager
and replayed from a CUDA graph; the time of one log point (`local_returns`: 468 reductions against one per-setting
launch); and the kernel launches per lock-step and per log point (`bsb_launch_count`).  The two variants are timed
in alternation, `rounds` times each, with CUDA events around `iters` calls after a warm-up; medians are reported.
The mnist experiments read synthetic idx files written to a temporary directory.  One JSON line per configuration,
then one with the card's name and power limit.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from bsuite_b200 import _lib, datasets, suite, sweep  # noqa: E402


def card():
  try:
    out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                         capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
  except (OSError, subprocess.SubprocessError, IndexError):
    out = 'nvidia-smi unavailable'
  return dict(torch_name=torch.cuda.get_device_name(), nvidia_smi=out)


def timed(fn, iters):
  """ms per call of `fn` over `iters` calls between CUDA events (after a synchronise)."""
  torch.cuda.synchronize()
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  e0.record()
  for _ in range(iters):
    fn()
  e1.record()
  torch.cuda.synchronize()
  return e0.elapsed_time(e1) / iters


def alternate(fns, iters, rounds):
  """Median ms per call of each of `fns`, timed in alternation."""
  samples = {k: [] for k in fns}
  for _ in range(rounds):
    for k, fn in fns.items():
      samples[k].append(timed(fn, iters))
  return {k: statistics.median(v) for k, v in samples.items()}


def launches(fn):
  lib = _lib.load()
  before = lib.bsb_launch_count()
  fn()
  torch.cuda.synchronize()
  return lib.bsb_launch_count() - before


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--lanes', type=int, nargs='+', default=[256, 1024])
  ap.add_argument('--steps', type=int, nargs='+', default=[1, 16])
  ap.add_argument('--iters', type=int, default=20)
  ap.add_argument('--rounds', type=int, default=5)
  args = ap.parse_args()
  if not torch.cuda.is_available():
    raise RuntimeError('bench_sweep_packed.py measures on a CUDA device; none is available')
  with tempfile.TemporaryDirectory() as tmp:
    os.environ[datasets.ENV_VAR] = datasets.write_synthetic_mnist(tmp, 4096, 16, 0)
    ids = list(sweep.SWEEP)
    for lanes in args.lanes:
      batches = dict(unpacked=suite.SweepBatch(ids, lanes=lanes, device='cuda', seed=0),
                     packed=suite.SweepBatch(ids, lanes=lanes, device='cuda', seed=0, packed=True))
      for name, batch in batches.items():
        batch.local_returns()
      log = alternate({k: b.local_returns for k, b in batches.items()}, args.iters, args.rounds)
      log_launches = {k: launches(b.local_returns) for k, b in batches.items()}
      for T in args.steps:
        for batch in batches.values():
          for _ in range(3):
            batch.rollout(T)
        eager = alternate({k: (lambda b=b: b.rollout(T)) for k, b in batches.items()}, args.iters, args.rounds)
        step_launches = {k: launches(lambda b=b: b.rollout(T)) for k, b in batches.items()}
        graphs = {k: b.capture(T) for k, b in batches.items()}
        for g in graphs.values():
          g.replay()
        graphed = alternate({k: g.replay for k, g in graphs.items()}, args.iters, args.rounds)
        del graphs
        row = dict(ids=len(ids), lanes_per_setting=lanes, T=T, handles={k: len(b.envs) for k, b in batches.items()},
                   eager_ms_per_lockstep=eager, graph_ms_per_lockstep=graphed,
                   eager_speedup=eager['unpacked'] / eager['packed'], graph_speedup=graphed['unpacked'] / graphed['packed'],
                   env_steps_per_s_eager={k: len(ids) * lanes * T / (v * 1e-3) for k, v in eager.items()},
                   launches_per_lockstep=step_launches, log_point_ms=log, log_point_launches=log_launches,
                   log_point_speedup=log['unpacked'] / log['packed'],
                   bytes_per_lockstep={k: b.bytes_per_step() * T for k, b in batches.items()})
        print(json.dumps(row), flush=True)
        for batch in batches.values():
          batch.set_ring(1)
      for batch in batches.values():
        batch.close()
      del batches
      torch.cuda.empty_cache()
  print(json.dumps(dict(card=card(), peak_mem_gb=torch.cuda.max_memory_allocated() / 1e9)), flush=True)


if __name__ == '__main__':
  main()
