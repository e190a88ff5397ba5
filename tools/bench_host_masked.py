#!/usr/bin/env python
"""Masked host-driven steps (`step_host(..., mask=...)`, bsb_step_host_masked) on one GPU.

    python tools/bench_host_masked.py [--out out/host_masked.jsonl] [--steps 200] [--warmup 20] [--repeats 5]

1. Time per decision.  Workloads: deep_sea N = 32 at B = 65 536, catch at B = 131 072 and cartpole at B = 131 072 (those
   of tools/bench_masked.py).  Variants: the unmasked `step_host`, masked `step_host` with a fixed random mask of 100 %,
   50 % and 1 % of the lanes (no budgets), and the route a host-side agent has without masked host steps: a device
   `step(mask=)` followed by `.cpu()` of reward, discount and step_type.  The `step_host` variants run waited on one
   handle and round-robin over two part handles (`wait=False`, one decision = one step of every part).  Actions and
   masks are pinned; every call ends with its scalars on the host, so the host clock around `--steps` calls times them.
2. Experiments run to a budget of `--episodes` episodes per lane by a host random policy (a pool of pinned action
   tensors): catch, bandit, deep_sea (ragged pack) and cartpole, each loaded as a pack of about 65 536 lanes.
   `run_episodes` (device masked steps) against `run_host_episodes`, and on the experiment's first id at the same
   batch `run_host_episodes` against `HostParts.run_episodes` with two parts.  Wall time per run, fresh handles each.

Variants alternate within each of `--repeats` windows; rows give the median (and range).  The card's name, power limit
and SM clocks are printed first.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import bsuite_b200  # noqa: E402
from bsuite_b200 import rollouts  # noqa: E402
from bsuite_b200 import sweep  # noqa: E402

WORKLOADS = (('deep_sea/11', 65536), ('catch/0', 131072), ('cartpole/0', 131072))
DENSITIES = (1.0, 0.5, 0.01)
EXPERIMENTS = ('catch', 'bandit', 'deep_sea', 'cartpole')
POOL = 8


def card():
  query = 'name,power.limit,clocks.max.sm,clocks.sm'
  out = subprocess.run(['nvidia-smi', f'--query-gpu={query}', '--format=csv,noheader'], capture_output=True, text=True)
  return dict(zip(query.split(','), [v.strip() for v in out.stdout.splitlines()[0].split(',')])) if out.stdout else {}


def pinned(tensor):
  return torch.empty(tensor.shape, dtype=tensor.dtype, pin_memory=True).copy_(tensor)


def action_pool(B, num_actions, seed):
  gen = torch.Generator().manual_seed(seed)
  return [pinned(torch.randint(0, num_actions, (B,), dtype=torch.int32, generator=gen)) for _ in range(POOL)]


def median_row(times, **fields):
  return dict(fields, median=round(statistics.median(times), 3), range=[round(min(times), 3), round(max(times), 3)])


def per_decision(args, bsuite_id, B):
  """Section 1 for one workload: {variant: [µs per decision, one per window]}."""
  env = bsuite_b200.load_from_id(bsuite_id, batch=B, device='cuda', seed=1)
  sizes = rollouts.split_sizes(B, 2)
  parts = [bsuite_b200.load_from_id(bsuite_id, batch=sizes[0], device='cuda', seed=1),
           bsuite_b200.load_from_id(bsuite_id, batch=sizes[1], device='cuda', seed=1, lane_offset=sizes[0])]
  actions = action_pool(B, env.num_actions, 0)
  gen = torch.Generator().manual_seed(1)
  masks = {d: pinned(torch.rand(B, generator=gen) < d) for d in DENSITIES}
  host, out = env.make_host_buffers(), env.make_buffers()
  env.reset(out=out)
  part_host = [p.make_host_buffers() for p in parts]
  part_out = [p.make_buffers() for p in parts]
  for p, o in zip(parts, part_out):
    p.reset(out=o)
  part_actions = [[a[:sizes[0]], a[sizes[0]:]] for a in actions]      # views of pinned memory stay pinned
  part_masks = {d: [m[:sizes[0]], m[sizes[0]:]] for d, m in masks.items()}
  dev_masks = {d: m.cuda() for d, m in masks.items()}

  def one(mask, n):
    for k in range(n):
      env.step_host(actions[k % POOL], host, out, mask=mask)

  def two(mask, n):
    for k in range(n):
      for i, p in enumerate(parts):
        if k:
          p.host_wait()
        p.step_host(part_actions[k % POOL][i], part_host[i], part_out[i], wait=False,
                    mask=None if mask is None else part_masks[mask][i])
    for p in parts:
      p.host_wait()

  def device_route(d, n):
    for k in range(n):
      ts = env.step(actions[k % POOL], out=out, mask=dev_masks[d])
      ts.reward.cpu(), ts.discount.cpu(), ts.step_type.cpu()

  variants = [('step_host', lambda n: one(None, n)), ('step_host 2 parts', lambda n: two(None, n))]
  for d in DENSITIES:
    variants += [(f'masked {d:.0%}', lambda n, d=d: one(masks[d], n)),
                 (f'masked {d:.0%} 2 parts', lambda n, d=d: two(d, n)),
                 (f'step(mask) {d:.0%} + .cpu()', lambda n, d=d: device_route(d, n))]
  for _, run in variants:
    run(args.warmup)
  torch.cuda.synchronize()
  times = {name: [] for name, _ in variants}
  for _ in range(args.repeats):
    for name, run in variants:
      torch.cuda.synchronize()
      start = time.perf_counter()
      run(args.steps)
      torch.cuda.synchronize()
      times[name].append((time.perf_counter() - start) * 1e6 / args.steps)
  for e in [env] + parts:
    e.close()
  return times


def to_budget(args, name, kind):
  """Section 2: wall seconds of one run of `kind` on fresh handles."""
  lanes = max(1, args.batch // len(sweep.BY_EXPERIMENT[name]))
  kw = dict(device='cuda', seed=2, track_episodes=True)
  if kind in ('run_episodes', 'run_host_episodes'):
    env = bsuite_b200.load_experiment(name, lanes, ragged=name == 'deep_sea', **kw)
  elif kind == 'id run_host_episodes':
    env = bsuite_b200.load_from_id(sweep.BY_EXPERIMENT[name][0], batch=lanes * len(sweep.BY_EXPERIMENT[name]), **kw)
  else:
    env = rollouts.HostParts(sweep.BY_EXPERIMENT[name][0], lanes * len(sweep.BY_EXPERIMENT[name]), parts=2, **kw)
  envs = env.envs if kind == 'HostParts' else [env]
  pools = [action_pool(e.batch, e.num_actions, 3) for e in envs]
  torch.cuda.synchronize()
  start = time.perf_counter()
  if kind == 'run_episodes':
    class Agent:
      calls = 0

      def select_action(self, timestep):
        del timestep
        self.calls += 1
        return pools[0][self.calls % POOL]

      def update(self, *unused):
        del unused
    rollouts.run_episodes(Agent(), env, args.episodes)
  elif kind == 'HostParts':
    env.run_episodes(lambda part, call, *unused: pools[part][call % POOL], args.episodes)
  else:
    rollouts.run_host_episodes(lambda call, *unused: pools[0][call % POOL], env, args.episodes)
  torch.cuda.synchronize()
  seconds = time.perf_counter() - start
  episodes = sum(float(e.episode_stats()['episode'].sum()) for e in envs)
  assert episodes == args.episodes * sum(e.batch for e in envs), (name, kind, episodes)
  env.close()
  return seconds


def main():
  parser = argparse.ArgumentParser()
  parser.add_argument('--out', default=None)
  parser.add_argument('--steps', type=int, default=200)
  parser.add_argument('--warmup', type=int, default=20)
  parser.add_argument('--repeats', type=int, default=5)
  parser.add_argument('--episodes', type=int, default=8)
  parser.add_argument('--batch', type=int, default=65536)
  args = parser.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit('bench_host_masked.py needs a CUDA device')
  rows = [dict(card=card())]
  print(json.dumps(rows[0]), flush=True)
  for bsuite_id, B in WORKLOADS:
    for variant, times in per_decision(args, bsuite_id, B).items():
      rows.append(median_row(times, section='per_decision', workload=bsuite_id, batch=B, variant=variant,
                             unit='us per decision'))
      print(json.dumps(rows[-1]), flush=True)
  kinds = ('run_episodes', 'run_host_episodes', 'id run_host_episodes', 'HostParts')
  for name in EXPERIMENTS:
    for kind in kinds:      # warm-up: module loading and every launch shape
      to_budget(args, name, kind)
    times = {kind: [] for kind in kinds}
    for _ in range(max(1, args.repeats // 2)):
      for kind in kinds:
        times[kind].append(to_budget(args, name, kind))
    for kind in kinds:
      rows.append(median_row(times[kind], section='to_budget', experiment=name, variant=kind, episodes=args.episodes,
                             unit='s per run'))
      print(json.dumps(rows[-1]), flush=True)
  if args.out:
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, 'w') as fh:
      for row in rows:
        fh.write(json.dumps(row) + '\n')


if __name__ == '__main__':
  main()
