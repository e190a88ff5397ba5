#!/usr/bin/env python
"""One ragged pack per experiment against one handle per setting: graph-captured rollouts on one GPU.

    python tools/bench_ragged.py [--out out/ragged.jsonl] [--lanes 256,4096] [--only deep_sea] [--replays 20]

For the four experiments whose settings differ in observation shape (deep_sea, deep_sea_stochastic, memory_size,
umbrella_distract), at each of `--lanes` lanes per setting and T = 1 and T = 64 steps per rollout:
  separate : one handle per setting, each rollout on a stream of its own (as SuiteBatch / SweepBatch run them)
  ragged   : one ragged pack of all settings (bsuite_b200.load_experiment(..., ragged=True)), the same lanes
both captured into one CUDA graph per variant (tools/bench_packed.py's `Captured`: actions sampled on the device,
observation buffers from `make_buffers`, so deep_sea's lie in compressible memory where the card has it) and
replayed, the two variants alternating.  Reported per row: µs per replay (median of `--repeats` windows, with the
range), kernel launches of one replay, env-steps/s and the algorithmic observation bytes/s (every element of every
observation written once, float32) beside the H100 SXM data-sheet HBM3 bandwidth of 3.35 TB/s.  The card's name and
power limit are printed first.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

import bsuite_b200  # noqa: E402
from tools.bench_packed import Captured  # noqa: E402

RAGGED = ('deep_sea', 'deep_sea_stochastic', 'memory_size', 'umbrella_distract')
HBM_BYTES_PER_S = 3.35e12


def compare(name, lanes, T, args):
  pack = bsuite_b200.load_experiment(name, lanes, device='cuda', seed=0, ragged=True)
  parts = [bsuite_b200.load_from_id(i, batch=lanes, device='cuda', seed=0) for i in pack.bsuite_ids]
  obs_bytes = T * lanes * 4 * sum(int(np.prod(shape)) for shape in pack.obs_shapes)
  variants = dict(separate=Captured(parts, T), ragged=Captured([pack], T))
  times = {k: [] for k in variants}
  for _ in range(args.repeats):
    for k, v in variants.items():
      times[k].append(v.time(args.replays))
  rows = []
  for k, v in variants.items():
    ts = sorted(times[k])
    dt = ts[len(ts) // 2]
    rows.append(dict(config=name, variant=k, lanes_per_setting=lanes, T=T, handles=len(v.envs), lanes=pack.batch,
                     launches_per_replay=v.launches, us_per_replay=dt * 1e6, us_range=[ts[0] * 1e6, ts[-1] * 1e6],
                     env_steps_per_s=T * pack.batch / dt, obs_bytes_per_replay=obs_bytes,
                     obs_bytes_per_s=obs_bytes / dt, obs_share_of_3_35_tb_s=obs_bytes / dt / HBM_BYTES_PER_S))
  del variants, pack, parts
  torch.cuda.empty_cache()
  return rows


def main():
  parser = argparse.ArgumentParser()
  parser.add_argument('--out', default=None)
  parser.add_argument('--lanes', default='256,4096')
  parser.add_argument('--only', default='')
  parser.add_argument('--replays', type=int, default=20)
  parser.add_argument('--repeats', type=int, default=3, help='timed windows per variant (median reported)')
  args = parser.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit('bench_ragged.py needs a CUDA device')
  card = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                        capture_output=True, text=True).stdout.strip().splitlines()
  print(json.dumps(dict(device=torch.cuda.get_device_name(0), nvidia_smi=card[:1])), flush=True)
  only = [s for s in args.only.split(',') if s]
  rows = []
  for name in RAGGED:
    if only and name not in only:
      continue
    for lanes in (int(s) for s in args.lanes.split(',')):
      for T in (1, 64):
        for row in compare(name, lanes, T, args):
          rows.append(row)
          print(json.dumps(row), flush=True)
  if args.out:
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, 'w') as f:
      for row in rows:
        f.write(json.dumps(row) + '\n')


if __name__ == '__main__':
  main()
