#!/usr/bin/env python
"""Agent loops to the episode budgets on one GPU: budgeted steps (`rollouts.run_episodes`, `SweepBatch.run_episodes`,
`SweepBatch.run_host_episodes`) against the loop `rollouts.run_episodes` used before them.

    python tools/bench_agent_episodes.py [--batches 64 4096 65536] [--episodes 5] [--lanes 64 1024]
                                         [--sweep-episodes 3] [--host-lanes 256]

(a) catch/0, deep_sea/0 and cartpole/0 at each batch size, `--episodes` episodes per lane, a device random agent
    (`rollouts.RandomAgent`, its own torch generator): wall time per call of `rollouts.run_episodes` and of the loop it
    replaced (`parent_run_episodes` below: four full-batch copies into a spare buffer set, a masked step and the LAST
    counting in torch per call), alternated `--rounds` times on fresh environments; medians.  Each round checks that
    both runs made the same number of calls and left the same bsuite_info(), episode statistics and log rows.
(b) The packed 468-id sweep at each `--lanes`, `--sweep-episodes` episodes per lane (None: every id's real budget),
    one RandomAgent per pack: wall time of `SweepBatch.run_episodes`, and of the parent loop driven pack by pack;
    per-setting sums compared bit for bit.
(c) `SweepBatch.run_host_episodes` on the packs of a few experiments at `--host-lanes` lanes, a random policy that
    writes numpy draws into a pinned tensor: wall time, against the same packs driven one after another by
    `rollouts.run_host_episodes`.

The mnist experiments read synthetic idx files written to a temporary directory.  One JSON line per measurement, then
one with the card's name and power limit.
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

import numpy as np  # noqa: E402
import torch  # noqa: E402

import bsuite_b200  # noqa: E402
from bsuite_b200 import datasets, rollouts, suite, sweep  # noqa: E402

HOST_IDS = [i for i in sweep.SWEEP if i.split('/')[0] in ('catch', 'deep_sea', 'bandit', 'memory_len', 'umbrella_length')]


def card():
  try:
    out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                         capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
  except (OSError, subprocess.SubprocessError, IndexError):
    out = 'nvidia-smi unavailable'
  return dict(torch_name=torch.cuda.get_device_name(), nvidia_smi=out)


def parent_run_episodes(agent, environment, num_episodes=None, check_every=16):
  """rollouts.run_episodes as it was before budgeted steps."""
  B, device = environment.batch, environment.device
  budget = rollouts.episode_budget(environment, num_episodes)
  finished = torch.zeros(B, dtype=torch.int64, device=device)
  active = budget > 0
  out = environment.make_buffers()
  timestep = environment.reset(out=out, mask=active)
  spare = environment.make_buffers()
  calls = 0
  while True:
    if calls % max(int(check_every), 1) == 0 and not bool(active.any()):
      return calls
    actions = agent.select_action(timestep)
    spare.observation.copy_(out.observation)
    spare.reward.copy_(out.reward)
    spare.discount.copy_(out.discount)
    spare.step_type.copy_(out.step_type)
    previous = spare.timestep()
    new_timestep = environment.step(actions, out=out, mask=active)
    calls += 1
    agent.update(previous, actions, new_timestep)
    finished += ((new_timestep.step_type == 2) & active).to(torch.int64)
    active = finished < budget
    timestep = new_timestep


def wall(fn):
  torch.cuda.synchronize()
  start = time.perf_counter()
  result = fn()
  torch.cuda.synchronize()
  return time.perf_counter() - start, result


def accumulators(env):
  acc = {f'info {k}': v for k, v in env.bsuite_info().items()}
  acc.update({f'stat {k}': v for k, v in env.episode_stats().items()})
  rows = env.logged_rows()
  acc['rows'], acc['counts'] = rows['rows'], rows['counts']
  return acc


def same(a, b):
  return a.keys() == b.keys() and all(torch.equal(a[k], b[k]) for k in a)


def one_environment(batches, episodes, rounds):
  for bsuite_id in ('catch/0', 'deep_sea/0', 'cartpole/0'):
    for batch in batches:
      samples = {'budgeted': [], 'parent': []}
      equal, calls = True, None
      for _ in range(rounds):
        got = {}
        for path, loop in (('budgeted', rollouts.run_episodes), ('parent', parent_run_episodes)):
          env = bsuite_b200.load_from_id(bsuite_id, batch=batch, device='cuda', seed=1, track_episodes=True,
                                         record_rows=True)
          agent = rollouts.RandomAgent(env.action_spec(), batch, device='cuda', seed=2)
          seconds, n = wall(lambda: loop(agent, env, num_episodes=episodes))
          samples[path].append(seconds / n)
          got[path] = (n, accumulators(env))
          env.close()
        equal = equal and got['budgeted'][0] == got['parent'][0] and same(got['budgeted'][1], got['parent'][1])
        calls = got['budgeted'][0]
      us = {k: statistics.median(v) * 1e6 for k, v in samples.items()}
      print(json.dumps(dict(part='a', bsuite_id=bsuite_id, batch=batch, num_episodes=episodes, calls=calls,
                            us_per_call=us, speedup=us['parent'] / us['budgeted'], bit_equal=equal)), flush=True)
      torch.cuda.empty_cache()


def sweep_agents(batch):
  return {k: rollouts.RandomAgent(env.action_spec(), env.batch, device='cuda', seed=i)
          for i, (k, env) in enumerate(batch.envs.items())}


def whole_sweep(lanes_list, episodes):
  for lanes in lanes_list:
    kw = dict(lanes=lanes, device='cuda', seed=0, record_rows=True, packed=True)
    batch = suite.SweepBatch(list(sweep.SWEEP), **kw)
    agents = sweep_agents(batch)
    seconds, calls = wall(lambda: batch.run_episodes(agents, num_episodes=episodes))
    driven = suite.SweepBatch(list(sweep.SWEEP), **kw)
    driven_agents = sweep_agents(driven)
    driven_seconds, driven_calls = wall(lambda: {k: parent_run_episodes(driven_agents[k], env, num_episodes=episodes)
                                                 for k, env in driven.envs.items()})
    steps = batch.local_returns()[:, 2].sum().item()
    print(json.dumps(dict(part='b', ids=len(batch.bsuite_ids), lanes=lanes, num_episodes=episodes,
                          max_calls=max(calls.values()), lane_steps=steps, seconds=seconds,
                          parent_driven_seconds=driven_seconds, speedup=driven_seconds / seconds,
                          bit_equal=calls == driven_calls and torch.equal(batch.local_returns(),
                                                                         driven.local_returns()))), flush=True)
    batch.close()
    driven.close()
    del batch, driven
    torch.cuda.empty_cache()


def host_policy(env, seed):
  rng = np.random.default_rng(seed)
  actions = torch.empty(env.batch, dtype=torch.int32, pin_memory=True)

  def policy(call, timestep, observation, mask):
    del call, timestep, observation, mask
    actions.numpy()[:] = rng.integers(0, env.num_actions, env.batch)
    return actions
  return policy


def host_sweep(lanes, episodes):
  kw = dict(lanes=lanes, device='cuda', seed=0, record_rows=True, packed=True)
  batch, driven = suite.SweepBatch(HOST_IDS, **kw), suite.SweepBatch(HOST_IDS, **kw)
  policies = {k: host_policy(env, i) for i, (k, env) in enumerate(batch.envs.items())}
  seconds, calls = wall(lambda: batch.run_host_episodes(policies, num_episodes=episodes))
  driven_seconds, driven_calls = wall(lambda: {k: rollouts.run_host_episodes(host_policy(env, i), env, episodes)
                                               for i, (k, env) in enumerate(driven.envs.items())})
  print(json.dumps(dict(part='c', ids=len(HOST_IDS), packs=list(batch.envs), lanes=lanes, num_episodes=episodes,
                        max_calls=max(calls.values()), seconds=seconds, one_after_another_seconds=driven_seconds,
                        speedup=driven_seconds / seconds,
                        bit_equal=calls == driven_calls and torch.equal(batch.local_returns(),
                                                                       driven.local_returns()))), flush=True)
  batch.close()
  driven.close()


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--batches', type=int, nargs='+', default=[64, 4096, 65536])
  ap.add_argument('--episodes', type=int, default=5)
  ap.add_argument('--rounds', type=int, default=3)
  ap.add_argument('--lanes', type=int, nargs='+', default=[64, 1024])
  ap.add_argument('--sweep-episodes', type=int, default=3, help='episodes per lane in (b); 0: every id\'s real budget')
  ap.add_argument('--host-lanes', type=int, default=256)
  ap.add_argument('--host-episodes', type=int, default=3)
  ap.add_argument('--skip', choices=['a', 'b', 'c'], nargs='*', default=[])
  args = ap.parse_args()
  if not torch.cuda.is_available():
    raise RuntimeError('bench_agent_episodes.py measures on a CUDA device; none is available')
  print(json.dumps(dict(card=card())), flush=True)
  with tempfile.TemporaryDirectory() as tmp:
    os.environ[datasets.ENV_VAR] = datasets.write_synthetic_mnist(tmp, 4096, 16, 0)
    if 'a' not in args.skip:
      one_environment(args.batches, args.episodes, args.rounds)
    if 'b' not in args.skip:
      whole_sweep(args.lanes, args.sweep_episodes or None)
    if 'c' not in args.skip:
      host_sweep(args.host_lanes, args.host_episodes)
  print(json.dumps(dict(card=card(), peak_mem_gb=torch.cuda.max_memory_allocated() / 1e9)), flush=True)


if __name__ == '__main__':
  main()
