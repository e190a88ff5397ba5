#!/usr/bin/env python
"""Masked rollouts (`rollout(..., mask=..., episodes_left=...)`, masked_kernel) on one GPU, in two legs.

    python tools/bench_masked_rollout.py [--out out/masked_rollout.jsonl] [--repeats 5] [--lanes 64] [--episodes 20]

Rollout cost: deep_sea N = 32 at B = 65 536 (observations in compressible memory, as make_buffers allocates them),
catch at B = 131 072 and cartpole at B = 131 072, the workloads of tools/bench_masked.py.  For each: `rollout(16)`, a
masked `rollout(16)` and 16 masked single steps, with fixed random masks of 100 %, 50 % and 1 % of the lanes and on-device
random actions (the masked steps take the same actions, sampled beforehand).  Every variant runs `--calls` launches
of 16 steps between CUDA events, the variants alternating within each of `--repeats` windows; reported per row: the
median µs per 16 steps (with the range) and active env-steps/s.

Run to budget: each of the 23 experiments, loaded with `load_experiment(name, --lanes, ragged=True,
record_rows=True)`, plays every setting's `bsuite_num_episodes`, capped at `--episodes`, once with
`rollouts.run_random_episodes` (64 steps per launch) and once with `rollouts.run_episodes` driven by an agent that
returns the host mirror of the on-device sampler (`random_actions(1, seed, first_step=steps_done)`), the two
alternating over `--repeats` windows on fresh environments.  Wall time ends in a device synchronise.  The two runs'
bsuite scores must be equal bit for bit (asserted) and are printed.  The card's name, SM clock and power limit are
printed first.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import bsuite_b200  # noqa: E402
from bsuite_b200 import analysis  # noqa: E402
from bsuite_b200 import datasets  # noqa: E402
from bsuite_b200 import rollouts  # noqa: E402
from bsuite_b200 import sweep  # noqa: E402

WORKLOADS = (('deep_sea/11', 65536), ('catch/0', 131072), ('cartpole/0', 131072))
DENSITIES = (1.0, 0.5, 0.01)
T = 16


def card():
  query = 'name,power.limit,clocks.max.sm,clocks.sm'
  out = subprocess.run(['nvidia-smi', f'--query-gpu={query}', '--format=csv,noheader'], capture_output=True, text=True)
  return dict(zip(query.split(','), [v.strip() for v in out.stdout.splitlines()[0].split(',')])) if out.stdout else {}


def rollout_cost(args, emit):
  for bsuite_id, B in WORKLOADS:
    env = bsuite_b200.load_from_id(bsuite_id, batch=B, device='cuda', seed=1)
    env.reset(out=env.make_buffers())
    out_t = env.make_buffers(T)
    out_1 = env.make_buffers()
    gen = torch.Generator(device='cuda').manual_seed(0)
    masks = {d: torch.rand(B, device='cuda', generator=gen) < d for d in DENSITIES}
    actions = torch.as_tensor(env.random_actions(T, 0, first_step=0)).to('cuda')

    def plain(n):
      for _ in range(n):
        env.rollout(T, out=out_t)

    def fused(mask):
      def run(n):
        for _ in range(n):
          env.rollout(T, out=out_t, mask=mask)
      return run

    def steps(mask):
      def run(n):
        for _ in range(n):
          for t in range(T):
            env.step(actions[t], out=out_1, mask=mask)
      return run

    variants = [('rollout(16)', None, plain)]
    for d in DENSITIES:
      variants += [(f'masked rollout(16) {int(d * 100)}%', masks[d], fused(masks[d])),
                   (f'16 masked steps {int(d * 100)}%', masks[d], steps(masks[d]))]
    for _, _, run in variants:
      run(args.warmup)
    torch.cuda.synchronize()
    times = {name: [] for name, _, _ in variants}
    for _ in range(args.repeats):
      for name, _, run in variants:
        start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        start.record()
        run(args.calls)
        stop.record()
        stop.synchronize()
        times[name].append(start.elapsed_time(stop) * 1e3 / args.calls)
    for name, mask, _ in variants:
      us = statistics.median(times[name])
      active = B if mask is None else int(mask.sum())
      emit(dict(leg='rollout cost', workload=bsuite_id, batch=B, variant=name, active_lanes=active,
                us_per_16_steps=round(us, 2), us_range=[round(min(times[name]), 2), round(max(times[name]), 2)],
                active_env_steps_per_s=active * T / (us * 1e-6)))
    env.close()


class StreamAgent:
  """The reference's random agent with the on-device sampler's actions, computed on the host."""

  def __init__(self, env, action_seed):
    self.env, self.action_seed = env, action_seed

  def select_action(self, timestep):
    del timestep
    return torch.as_tensor(self.env.random_actions(1, self.action_seed, first_step=self.env.steps_done)[0]).to('cuda')

  def update(self, timestep, action, new_timestep):
    del timestep, action, new_timestep


def run_to_budget(args, emit):
  action_seed = 7
  if not os.environ.get(datasets.ENV_VAR):      # mnist's settings: synthetic idx files outside the tree
    os.environ[datasets.ENV_VAR] = datasets.write_synthetic_mnist(tempfile.mkdtemp(prefix='bsb_mnist_'), 256, 16, 0)
  for name in sorted(sweep.BY_EXPERIMENT):
    def fresh():
      return bsuite_b200.load_experiment(name, args.lanes, device='cuda', seed=3, track_episodes=True,
                                         record_rows=True, ragged=True)
    probe = fresh()
    budgets = [min(spec.bsuite_num_episodes, args.episodes) for spec in probe._pack[1]]
    probe.close()

    def run(kind):
      env = fresh()
      specs = env._pack[1]
      saved = [spec.bsuite_num_episodes for spec in specs]
      for spec, n in zip(specs, budgets):      # the capped budgets, lowered in place for this run
        spec.bsuite_num_episodes = n
      try:
        torch.cuda.synchronize()
        start = time.perf_counter()
        if kind == 'fused':
          calls = rollouts.run_random_episodes(env, action_seed=action_seed, steps_per_launch=64)
        else:
          calls = rollouts.run_episodes(StreamAgent(env, action_seed), env)
        torch.cuda.synchronize()
        seconds = time.perf_counter() - start
      finally:
        for spec, n in zip(specs, saved):
          spec.bsuite_num_episodes = n
      score = analysis.bsuite_score(env).score[analysis.EXPERIMENTS.index(name)].cpu()
      env.close()
      return seconds, calls, score

    times = {'fused': [], 'stepped': []}
    scores, calls = {}, {}
    for _ in range(args.repeats):
      for kind in times:
        seconds, calls[kind], scores[kind] = run(kind)
        times[kind].append(seconds)
    assert torch.equal(scores['fused'].view(torch.int64), scores['stepped'].view(torch.int64)), name
    fused, stepped = statistics.median(times['fused']), statistics.median(times['stepped'])
    emit(dict(leg='run to budget', experiment=name, lanes_per_setting=args.lanes, settings=len(budgets),
              episodes=budgets, calls_fused=calls['fused'], calls_stepped=calls['stepped'],
              s_run_random_episodes=round(fused, 4), s_run_episodes=round(stepped, 4),
              speedup=round(stepped / fused, 2), mean_score=float(scores['fused'].mean())))


def main():
  parser = argparse.ArgumentParser()
  parser.add_argument('--out', default=None)
  parser.add_argument('--calls', type=int, default=50, help='launches of 16 steps per timed window (rollout cost)')
  parser.add_argument('--warmup', type=int, default=5)
  parser.add_argument('--repeats', type=int, default=5)
  parser.add_argument('--lanes', type=int, default=64, help='lanes per setting (run to budget)')
  parser.add_argument('--episodes', type=int, default=20, help='episode cap per setting (run to budget)')
  parser.add_argument('--legs', default='cost,budget')
  args = parser.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit('bench_masked_rollout.py needs a CUDA device')
  rows = []

  def emit(row):
    rows.append(row)
    print(json.dumps(row), flush=True)

  emit(dict(card=card()))
  legs = args.legs.split(',')
  if 'cost' in legs:
    rollout_cost(args, emit)
  if 'budget' in legs:
    run_to_budget(args, emit)
  if args.out:
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, 'w') as fh:
      for row in rows:
        fh.write(json.dumps(row) + '\n')


if __name__ == '__main__':
  main()
