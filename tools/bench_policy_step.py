#!/usr/bin/env python
"""Action selection inside the budgeted step (`select_policy`, `bsb_step_budgeted_policy`) against the same rule in
torch (`select_action`), for an agent with a reference-sized DQN network.

    python tools/bench_policy_step.py [--batches 64 1024 4096 65536] [--episodes 5] [--rounds 3] [--lanes 64]
                                      [--sweep-episodes 3] [--rules epsilon_greedy softmax]

The network is the reference dqn's MLP (baselines/jax/dqn: two hidden layers of 50, ReLU) with fixed random weights,
over the flattened observation.  Per rule, two agents share it:
  torch   `select_action`: the rule as a chain of torch kernels -- epsilon-greedy: rand, compare, randint, max, eq, a
          random argmax among the maxima (uniform noise on the tied entries) and where; softmax: multinomial over
          softmax(logits).
  policy  `select_policy`: `rollouts.EpsilonGreedy(q, 0.1)` / `rollouts.Softmax(q)`, chosen inside the step.
(a) catch/0, deep_sea/0 and cartpole/0 at each batch size, `--episodes` episodes per lane: wall time per call of
    `rollouts.run_episodes`, the two agents alternated `--rounds` times on fresh environments; medians.
(b) The packed 468-id sweep at each `--lanes`, `--sweep-episodes` episodes per lane, one network per pack (a ragged
    pack's observations zero-padded to its largest setting): wall time of `SweepBatch.run_episodes` per lock-step.
The two agents draw different random numbers, so their runs differ; each row reports both call counts.  The mnist
experiments read synthetic idx files written to a temporary directory.  One JSON line per measurement, then one with
the card's name and power limit.
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
from bsuite_b200 import datasets, rollouts, suite, sweep  # noqa: E402

EPSILON = 0.1


def card():
  try:
    out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                         capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
  except (OSError, subprocess.SubprocessError, IndexError):
    out = 'nvidia-smi unavailable'
  return dict(torch_name=torch.cuda.get_device_name(), nvidia_smi=out)


class Network:
  """dqn's MLP [in, 50, 50, A] with fixed random weights over the zero-padded, flattened observation."""

  def __init__(self, env, seed):
    self.env = env
    g = torch.Generator().manual_seed(seed)
    parts = env.split_observation(env.make_buffers().observation)
    self.size = max(int(p[0].numel()) for p in parts)
    sizes = [self.size, 50, 50, env.num_actions]
    self.layers = [((torch.randn(a, b, generator=g) / a ** 0.5).cuda(), torch.zeros(b, device='cuda'))
                   for a, b in zip(sizes[:-1], sizes[1:])]

  def __call__(self, observation):
    parts = [p.reshape(p.shape[0], -1).float() for p in self.env.split_observation(observation)]
    x = torch.cat([torch.nn.functional.pad(p, (0, self.size - p.shape[1])) for p in parts])
    for k, (w, b) in enumerate(self.layers):
      x = torch.addmm(b, x, w)
      if k + 1 < len(self.layers):
        x = torch.relu(x)
    return x.contiguous()


class TorchAgent:
  def __init__(self, env, rule, seed):
    self.net, self.rule, self.B, self.A = Network(env, seed), rule, env.batch, env.num_actions
    self.gen = torch.Generator(device='cuda').manual_seed(seed)

  def select_action(self, timestep):
    q = self.net(timestep.observation)
    if self.rule == 'softmax':
      return torch.multinomial(torch.softmax(q, 1), 1, generator=self.gen).view(-1).int()
    explore = torch.rand(self.B, device='cuda', generator=self.gen) < EPSILON
    uniform = torch.randint(0, self.A, (self.B,), device='cuda', generator=self.gen)
    ties = q == q.max(1, keepdim=True).values
    noise = torch.rand(self.B, self.A, device='cuda', generator=self.gen)
    greedy = torch.where(ties, noise, -1.0).argmax(1)
    return torch.where(explore, uniform, greedy).int()

  def update(self, timestep, actions, new_timestep):
    del timestep, actions, new_timestep


class PolicyAgent:
  def __init__(self, env, rule, seed):
    self.net, self.rule = Network(env, seed), rule

  def select_policy(self, timestep):
    q = self.net(timestep.observation)
    return rollouts.Softmax(q) if self.rule == 'softmax' else rollouts.EpsilonGreedy(q, EPSILON)

  def update(self, timestep, actions, new_timestep):
    del timestep, actions, new_timestep


AGENTS = {'torch': TorchAgent, 'policy': PolicyAgent}


def wall(fn):
  torch.cuda.synchronize()
  start = time.perf_counter()
  result = fn()
  torch.cuda.synchronize()
  return time.perf_counter() - start, result


def one_environment(rule, batches, episodes, rounds):
  for bsuite_id in ('catch/0', 'deep_sea/0', 'cartpole/0'):
    for batch in batches:
      samples, calls = {k: [] for k in AGENTS}, {}
      for _ in range(rounds):
        for name, make in AGENTS.items():
          env = bsuite_b200.load_from_id(bsuite_id, batch=batch, device='cuda', seed=1, track_episodes=True,
                                         record_rows=True)
          agent = make(env, rule, 2)
          seconds, n = wall(lambda: rollouts.run_episodes(agent, env, num_episodes=episodes, policy_seed=3))
          samples[name].append(seconds / n)
          calls[name] = n
          env.close()
      us = {k: statistics.median(v) * 1e6 for k, v in samples.items()}
      print(json.dumps(dict(part='a', rule=rule, bsuite_id=bsuite_id, batch=batch, num_episodes=episodes, calls=calls,
                            us_per_call=us, speedup=us['torch'] / us['policy'])), flush=True)
      torch.cuda.empty_cache()


def whole_sweep(rule, lanes_list, episodes, rounds):
  for lanes in lanes_list:
    samples, calls = {k: [] for k in AGENTS}, {}
    for _ in range(rounds):
      for name, make in AGENTS.items():
        batch = suite.SweepBatch(list(sweep.SWEEP), lanes=lanes, device='cuda', seed=0, record_rows=True, packed=True)
        agents = {k: make(env, rule, i) for i, (k, env) in enumerate(batch.envs.items())}
        seconds, n = wall(lambda: batch.run_episodes(agents, num_episodes=episodes, policy_seed=3))
        lock_steps = max(n.values())
        samples[name].append(seconds / lock_steps)
        calls[name] = lock_steps
        batch.close()
        del batch, agents
        torch.cuda.empty_cache()
    us = {k: statistics.median(v) * 1e6 for k, v in samples.items()}
    print(json.dumps(dict(part='b', rule=rule, ids=len(sweep.SWEEP), lanes=lanes, num_episodes=episodes,
                          lock_steps=calls, us_per_lock_step=us, speedup=us['torch'] / us['policy'])), flush=True)


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--batches', type=int, nargs='+', default=[64, 1024, 4096, 65536])
  ap.add_argument('--episodes', type=int, default=5)
  ap.add_argument('--rounds', type=int, default=3)
  ap.add_argument('--lanes', type=int, nargs='+', default=[64])
  ap.add_argument('--sweep-episodes', type=int, default=3)
  ap.add_argument('--rules', nargs='+', default=['epsilon_greedy', 'softmax'], choices=['epsilon_greedy', 'softmax'])
  ap.add_argument('--skip', choices=['a', 'b'], nargs='*', default=[])
  args = ap.parse_args()
  if not torch.cuda.is_available():
    raise RuntimeError('bench_policy_step.py measures on a CUDA device; none is available')
  print(json.dumps(dict(card=card())), flush=True)
  with tempfile.TemporaryDirectory() as tmp:
    os.environ[datasets.ENV_VAR] = datasets.write_synthetic_mnist(tmp, 4096, 16, 0)
    for rule in args.rules:
      if 'a' not in args.skip:
        one_environment(rule, args.batches, args.episodes, args.rounds)
      if 'b' not in args.skip:
        whole_sweep(rule, args.lanes, args.sweep_episodes, args.rounds)
  print(json.dumps(dict(card=card(), peak_mem_gb=torch.cuda.max_memory_allocated() / 1e9)), flush=True)


if __name__ == '__main__':
  main()
