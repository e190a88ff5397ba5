#!/usr/bin/env python
"""Masked steps (`step(..., mask=...)`, masked_kernel) against the plain `step` on one GPU.

    python tools/bench_masked.py [--out out/masked.jsonl] [--steps 200] [--warmup 20] [--repeats 5]

Workloads: deep_sea N = 32 at B = 65 536 (observations in compressible memory, as make_buffers allocates them),
catch at B = 131 072 and cartpole at B = 131 072.  For each: the plain step, and masked steps whose mask selects
100 %, 50 % and 1 % of the lanes (a fixed random mask).  Every variant runs `--steps` calls between CUDA events, the
variants alternating within each of `--repeats` windows; reported per row: the median µs per call (with the range),
active env-steps/s (active lanes / time) and the algorithmic bytes per active lane (suite.algorithmic_bytes_per_lane_step
plus one mask byte for masked calls).  The card's name, SM clock and power limit are printed first.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import bsuite_b200  # noqa: E402
from bsuite_b200 import suite  # noqa: E402

WORKLOADS = (('deep_sea/11', 65536), ('catch/0', 131072), ('cartpole/0', 131072))
DENSITIES = (1.0, 0.5, 0.01)


def card():
  query = 'name,power.limit,clocks.max.sm,clocks.sm'
  out = subprocess.run(['nvidia-smi', f'--query-gpu={query}', '--format=csv,noheader'], capture_output=True, text=True)
  return dict(zip(query.split(','), [v.strip() for v in out.stdout.splitlines()[0].split(',')])) if out.stdout else {}


def main():
  parser = argparse.ArgumentParser()
  parser.add_argument('--out', default=None)
  parser.add_argument('--steps', type=int, default=200)
  parser.add_argument('--warmup', type=int, default=20)
  parser.add_argument('--repeats', type=int, default=5)
  args = parser.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit('bench_masked.py needs a CUDA device')
  print(json.dumps(dict(card=card())), flush=True)
  rows = []
  for bsuite_id, B in WORKLOADS:
    env = bsuite_b200.load_from_id(bsuite_id, batch=B, device='cuda', seed=1)
    out = env.make_buffers()
    env.reset(out=out)
    gen = torch.Generator(device='cuda').manual_seed(0)
    actions = [torch.randint(0, env.num_actions, (B,), dtype=torch.int32, device='cuda', generator=gen)
               for _ in range(8)]
    masks = {d: torch.rand(B, device='cuda', generator=gen) < d for d in DENSITIES}
    variants = [('plain', None)] + [(f'masked {int(d * 100)}%', masks[d]) for d in DENSITIES]

    def run(mask, n):
      for k in range(n):
        if mask is None:
          env.step(actions[k % 8], out=out)
        else:
          env.step(actions[k % 8], out=out, mask=mask)

    for _, mask in variants:
      run(mask, args.warmup)
    torch.cuda.synchronize()
    times = {name: [] for name, _ in variants}
    for _ in range(args.repeats):
      for name, mask in variants:
        start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        start.record()
        run(mask, args.steps)
        stop.record()
        stop.synchronize()
        times[name].append(start.elapsed_time(stop) * 1e3 / args.steps)
    per_lane = suite.algorithmic_bytes_per_lane_step(env)
    for name, mask in variants:
      us = statistics.median(times[name])
      active = B if mask is None else int(mask.sum())
      row = dict(workload=bsuite_id, batch=B, variant=name, active_lanes=active, us_per_call=round(us, 2),
                 us_range=[round(min(times[name]), 2), round(max(times[name]), 2)],
                 active_env_steps_per_s=active / (us * 1e-6),
                 bytes_per_active_lane=per_lane + (0 if mask is None else 1))
      rows.append(row)
      print(json.dumps(row), flush=True)
    env.close()
  if args.out:
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, 'w') as fh:
      for row in rows:
        fh.write(json.dumps(row) + '\n')


if __name__ == '__main__':
  main()
