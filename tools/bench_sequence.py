#!/usr/bin/env python
"""Per-lane sequence buffers filled inside the budgeted step (`LaneSequence`, `bsb_step_budgeted_sequence`), against
the same buffers kept by the agent in torch.

    python tools/bench_sequence.py [--batches 64 1024 4096 65536] [--episodes 3] [--rounds 3] [--length 32]
                                   [--lanes 64] [--sweep-episodes 2]

Both agents share one network (the reference actor_critic's: an MLP torso [64, 64] with ReLU, a policy head and a
value head, fixed random weights, in torch) and one rule (softmax over the policy head, chosen inside the step with
the same policy seed), so they play the same transitions.  Neither does SGD: only the buffer cost is compared.
  torch     keeps per-lane windows of `--length` transitions in `update` with torch ops, as sequence.py's Buffer
            per lane -- the restart test, the first observation, five scatter-with-where writes, the length and the
            ready flag.
  sequence  carries a `LaneSequence` (`agent.sequence`), so `run_episodes` fills every window in the step.
(a) catch/0, deep_sea/0 and cartpole/0 at each batch size, `--episodes` episodes per lane: wall time per call of
    `rollouts.run_episodes`, the two agents alternated `--rounds` times on fresh environments; medians.  The buffers,
    lengths and ready flags the two agents left are compared and reported bit-equal or not, with both call counts.
(b) The packed 468-id sweep at `--lanes` lanes per id: wall time of `SweepBatch.run_episodes` per lock-step.  The
    mnist experiments read synthetic idx files written to a temporary directory.  One JSON line per measurement, then
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

import torch  # noqa: E402

import bsuite_b200  # noqa: E402
from bsuite_b200 import datasets, rollouts, suite, sweep  # noqa: E402

POLICY_SEED = 5
FIELDS = ('actions', 'rewards', 'discounts', 'step_types', 'length', 'ready')


def card():
  try:
    out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                         capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
  except (OSError, subprocess.SubprocessError, IndexError):
    out = 'nvidia-smi unavailable'
  return dict(torch_name=torch.cuda.get_device_name(), nvidia_smi=out)


class Network:
  """actor_critic's network: torso [in, 64, 64] with ReLU over the zero-padded, flattened observation, then a policy
  head [64, A] and a value head [64, 1]; fixed random weights."""

  def __init__(self, env, seed):
    self.env = env
    g = torch.Generator().manual_seed(seed)
    parts = env.split_observation(env.make_buffers().observation)
    self.size = max(int(p[0].numel()) for p in parts)

    def layer(a, b):
      return (torch.randn(a, b, generator=g) / a ** 0.5).cuda(), torch.zeros(b, device='cuda')
    self.torso = [layer(self.size, 64), layer(64, 64)]
    self.policy, self.value = layer(64, env.num_actions), layer(64, 1)

  def __call__(self, observation):
    parts = [p.reshape(p.shape[0], -1).float() for p in self.env.split_observation(observation)]
    x = torch.cat([torch.nn.functional.pad(p, (0, self.size - p.shape[1])) for p in parts])
    for w, b in self.torso:
      x = torch.relu(torch.addmm(b, x, w))
    logits = torch.addmm(self.policy[1], x, self.policy[0]).contiguous()
    value = torch.addmm(self.value[1], x, self.value[0]).squeeze(-1)
    return logits, value


class SequenceAgent:
  def __init__(self, env, seed, T):
    self.net = Network(env, seed)
    self.sequence = rollouts.LaneSequence(env, T)

  def select_policy(self, timestep):
    logits, _ = self.net(timestep.observation)
    return rollouts.Softmax(logits)

  def update(self, timestep, actions, new_timestep):
    pass


class TorchAgent(SequenceAgent):
  """The same buffers kept in `update` with torch ops (LaneSequence's layout, so the two compare whole)."""

  def __init__(self, env, seed, T, budget):
    self.env, self.net, self.T, self.budget = env, Network(env, seed), T, budget
    B = env.batch
    self.lanes = torch.arange(B, device='cuda')
    self.lasts = torch.zeros(B, dtype=torch.int64, device='cuda')
    obs = env.make_buffers().observation
    # observations per part: the whole [B, ...] tensor, or each setting's [L, ...] view of a ragged pack
    self.observations = [torch.zeros((T + 1,) + tuple(p.shape), dtype=p.dtype, device='cuda') for p in self._split(obs)]
    self.actions = torch.zeros((T, B), dtype=torch.int32, device='cuda')
    self.rewards = torch.zeros((T, B), dtype=torch.float32, device='cuda')
    self.discounts = torch.zeros((T, B), dtype=torch.float32, device='cuda')
    self.step_types = torch.zeros((T, B), dtype=torch.int32, device='cuda')
    self.length = torch.zeros(B, dtype=torch.int64, device='cuda')
    self.ready = torch.zeros(B, dtype=torch.bool, device='cuda')

  def _split(self, obs):
    return self.env.split_observation(obs) if self.env.ragged else (obs,)

  def update(self, timestep, actions, new_timestep):
    T = self.T
    stepped = self.lasts < self.budget
    app = stepped & (new_timestep.step_type != 0)
    t = self.length
    before = self.step_types.gather(0, (t - 1).clamp(min=0).unsqueeze(0)).squeeze(0)
    t = torch.where((t == T) | ((t > 0) & (before == 2)), torch.zeros_like(t), t)
    L = self.env.lanes_per_setting
    for k, (seq, o_tm1, o_t) in enumerate(zip(self.observations, self._split(timestep.observation),
                                              self._split(new_timestep.observation))):
      lanes = slice(k * L, (k + 1) * L) if self.env.ragged else slice(None)
      a, tk, idx = app[lanes], t[lanes], self.lanes[:o_t.shape[0]]
      shape = (-1,) + (1,) * (o_t.dim() - 1)
      seq[0] = torch.where((a & (tk == 0)).view(shape), o_tm1, seq[0])
      seq[tk + 1, idx] = torch.where(a.view(shape), o_t, seq[tk + 1, idx])
    for buf, value in ((self.actions, actions), (self.rewards, new_timestep.reward),
                       (self.discounts, new_timestep.discount), (self.step_types, new_timestep.step_type)):
      buf[t, self.lanes] = torch.where(app, value.to(buf.dtype), buf[t, self.lanes])
    self.length = torch.where(app, t + 1, self.length)
    self.ready = app & ((t + 1 == T) | (new_timestep.step_type == 2))
    self.lasts += ((new_timestep.step_type == 2) & stepped).to(torch.int64)


def same_buffers(torch_agent, sequence_agent):
  s, env = sequence_agent.sequence, torch_agent.env
  parts = env.split_observation(s.observations) if env.ragged else (s.observations,)
  pairs = list(zip(torch_agent.observations, parts)) + [(getattr(torch_agent, f), getattr(s, f)) for f in FIELDS]
  return all(torch.equal(a, b) for a, b in pairs)


def wall(fn):
  torch.cuda.synchronize()
  t0 = time.perf_counter()
  out = fn()
  torch.cuda.synchronize()
  return time.perf_counter() - t0, out


def one_environment(bsuite_id, B, episodes, rounds, T):
  times = {'torch': [], 'sequence': []}
  equal, calls = True, {'torch': [], 'sequence': []}
  for r in range(rounds):
    for kind in (('torch', 'sequence') if r % 2 == 0 else ('sequence', 'torch')):
      env = bsuite_b200.load_from_id(bsuite_id, batch=B, device='cuda', seed=1 + r)
      agent = TorchAgent(env, 3, T, episodes) if kind == 'torch' else SequenceAgent(env, 3, T)
      seconds, n = wall(lambda: rollouts.run_episodes(agent, env, num_episodes=episodes, policy_seed=POLICY_SEED))
      times[kind].append(seconds / n * 1e6)
      calls[kind].append(n)
      if kind == 'torch':
        torch_agent = agent
      else:
        sequence_agent = agent
    equal = equal and same_buffers(torch_agent, sequence_agent)
    del torch_agent, sequence_agent
  t, q = statistics.median(times['torch']), statistics.median(times['sequence'])
  print(json.dumps(dict(case='run_episodes', bsuite_id=bsuite_id, batch=B, max_sequence_length=T, episodes=episodes,
                        torch_us_per_call=round(t, 1), sequence_us_per_call=round(q, 1), speedup=round(t / q, 2),
                        calls=calls, calls_equal=calls['torch'] == calls['sequence'], buffers_bit_equal=equal)),
        flush=True)


def whole_sweep(lanes, T, episodes, rounds):
  times = {'torch': [], 'sequence': []}
  equal, lock_steps = True, {}
  for r in range(rounds):
    for kind in (('torch', 'sequence') if r % 2 == 0 else ('sequence', 'torch')):
      batch = suite.SweepBatch(sweep.SWEEP, lanes=lanes, device='cuda', seed=2 + r, packed=True)
      if kind == 'torch':
        agents = {k: TorchAgent(env, i, T, episodes) for i, (k, env) in enumerate(batch.envs.items())}
      else:
        agents = {k: SequenceAgent(env, i, T) for i, (k, env) in enumerate(batch.envs.items())}
      seconds, calls = wall(lambda: batch.run_episodes(agents, num_episodes=episodes, policy_seed=POLICY_SEED))
      times[kind].append(seconds / max(calls.values()) * 1e6)
      lock_steps[kind] = calls
      if kind == 'torch':
        torch_agents = agents
      else:
        sequence_agents = agents
      batch.close()
    equal = equal and all(same_buffers(torch_agents[k], sequence_agents[k]) for k in torch_agents)
  t, q = statistics.median(times['torch']), statistics.median(times['sequence'])
  print(json.dumps(dict(case='sweep', packs=len(torch_agents), lanes=lanes, max_sequence_length=T, episodes=episodes,
                        lock_steps=max(lock_steps['sequence'].values()),
                        calls_equal=lock_steps['torch'] == lock_steps['sequence'],
                        torch_us_per_lock_step=round(t, 1), sequence_us_per_lock_step=round(q, 1),
                        speedup=round(t / q, 2), buffers_bit_equal=equal)), flush=True)


def main():
  p = argparse.ArgumentParser()
  p.add_argument('--batches', type=int, nargs='+', default=[64, 1024, 4096, 65536])
  p.add_argument('--ids', nargs='+', default=['catch/0', 'deep_sea/0', 'cartpole/0'])
  p.add_argument('--episodes', type=int, default=3)
  p.add_argument('--rounds', type=int, default=3)
  p.add_argument('--length', type=int, default=32)
  p.add_argument('--lanes', type=int, default=64)
  p.add_argument('--sweep-episodes', type=int, default=2)
  p.add_argument('--sweep-rounds', type=int, default=1)
  args = p.parse_args()
  with tempfile.TemporaryDirectory() as tmp:
    os.environ[datasets.ENV_VAR] = datasets.write_synthetic_mnist(tmp, 4096, 16, 0)
    for bsuite_id in args.ids:
      for B in args.batches:
        one_environment(bsuite_id, B, args.episodes, args.rounds, args.length)
    if args.lanes > 0:
      whole_sweep(args.lanes, args.length, args.sweep_episodes, args.sweep_rounds)
  print(json.dumps(dict(card=card())), flush=True)


if __name__ == '__main__':
  main()
