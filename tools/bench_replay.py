#!/usr/bin/env python
"""Per-lane replay recorded inside the budgeted step (`LaneReplay`, `bsb_step_budgeted_record`) and sampled on the
device (`LaneReplay.sample`, `bsb_replay_sample`), against the same rings kept by the agent in torch.

    python tools/bench_replay.py [--batches 64 1024 4096] [--episodes 3] [--rounds 3] [--sample 32]
                                 [--ring-bytes 2e9] [--lanes 64] [--sweep-capacity 16] [--sweep-episodes 2]

Both agents share one network (the reference dqn's MLP: two hidden layers of 50, ReLU, fixed random weights) and one
rule (epsilon-greedy, 0.1, chosen inside the step with the same policy seed), so they play the same transitions:
  torch   keeps per-lane rings in `update` with torch ops -- the keep mask (stepped and not FIRST), per-lane slots,
          five scatter-with-where writes and the count -- and samples `--sample` transitions per lane with
          `torch.randint` and five gathers.
  record  carries a `LaneReplay` (`agent.replay`), so `run_episodes` records every transition in the step, and
          samples with `LaneReplay.sample(--sample)`.
(a) catch/0, deep_sea/0 and cartpole/0 at each batch size, `--episodes` episodes per lane, the capacity the largest
    power of two up to 10 000 whose rings fit in `--ring-bytes`: wall time per call of `rollouts.run_episodes`, the
    two agents alternated `--rounds` times on fresh environments; medians.  The rings the two agents filled are
    compared and reported bit-equal or not.  The sample kernel alone is timed with CUDA events on the filled rings,
    and its achieved bandwidth is computed from its algorithmic bytes (every sampled row and scalar read once from
    the ring and written once to the batch, plus the per-lane counts) against 3.35 TB/s.
(b) The packed 468-id sweep at `--lanes` lanes per id with `--sweep-capacity` slots: wall time of
    `SweepBatch.run_episodes` per lock-step.  The mnist experiments read synthetic idx files written to a temporary
    directory.  One JSON line per measurement, then one with the card's name and power limit.
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

EPSILON, POLICY_SEED, HBM = 0.1, 5, 3.35e12


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
  """Per-lane rings kept in `update` with torch ops, sampled with torch.randint and gathers."""

  def __init__(self, env, seed, capacity, budget, sample):
    self.env, self.net, self.capacity, self.sample = env, Network(env, seed), capacity, sample
    B = env.batch
    self.lanes = torch.arange(B, device='cuda')
    self.budget = budget
    self.lasts = torch.zeros(B, dtype=torch.int64, device='cuda')
    self.num_added = torch.zeros(B, dtype=torch.int64, device='cuda')
    self.gen = torch.Generator(device='cuda').manual_seed(seed)
    obs = env.make_buffers().observation
    # observations per part: the whole [B, ...] tensor, or each setting's [L, ...] view of a ragged pack
    self.parts = env.ragged
    self.obs_tm1 = [torch.zeros((capacity,) + tuple(p.shape), dtype=p.dtype, device='cuda') for p in self._split(obs)]
    self.obs = [torch.zeros_like(x) for x in self.obs_tm1]
    self.actions = torch.zeros((capacity, B), dtype=torch.int32, device='cuda')
    self.reward = torch.zeros((capacity, B), dtype=torch.float32, device='cuda')
    self.discount = torch.zeros((capacity, B), dtype=torch.float32, device='cuda')
    self.batch = None

  def _split(self, obs):
    return self.env.split_observation(obs) if self.parts else (obs,)

  def select_policy(self, timestep):
    return rollouts.EpsilonGreedy(self.net(timestep.observation), EPSILON)

  def update(self, timestep, actions, new_timestep):
    stepped = self.lasts < self.budget
    keep = stepped & (new_timestep.step_type != 0)
    slot = self.num_added % self.capacity
    L = self.env.lanes_per_setting
    for k, (ring_tm1, ring, o_tm1, o_t) in enumerate(zip(self.obs_tm1, self.obs, self._split(timestep.observation),
                                                         self._split(new_timestep.observation))):
      lanes = slice(k * L, (k + 1) * L) if self.parts else slice(None)
      s, kp, idx = slot[lanes], keep[lanes], self.lanes[:o_t.shape[0]]
      shape = (-1,) + (1,) * (o_t.dim() - 1)
      ring_tm1[s, idx] = torch.where(kp.view(shape), o_tm1, ring_tm1[s, idx])
      ring[s, idx] = torch.where(kp.view(shape), o_t, ring[s, idx])
    for ring, value in ((self.actions, actions), (self.reward, new_timestep.reward),
                        (self.discount, new_timestep.discount)):
      ring[slot, self.lanes] = torch.where(keep, value.to(ring.dtype), ring[slot, self.lanes])
    self.num_added += keep.to(torch.int64)
    self.lasts += ((new_timestep.step_type == 2) & stepped).to(torch.int64)
    # a minibatch per lane from its filled slots (a lane with none draws slot 0, which holds zeros)
    n = self.num_added.clamp(1, self.capacity)
    idx = torch.randint(0, 1 << 62, (self.sample, self.env.batch), device='cuda', generator=self.gen) % n
    self.batch = [ring[idx, self.lanes] for ring in (self.actions, self.reward, self.discount)]
    for k, (ring_tm1, ring) in enumerate(zip(self.obs_tm1, self.obs)):
      lanes = slice(k * L, (k + 1) * L) if self.parts else slice(None)
      part = idx[:, lanes]
      rows = self.lanes[:ring.shape[1]]
      self.batch += [ring_tm1[part, rows], ring[part, rows]]


class RecordAgent:
  def __init__(self, env, seed, capacity, sample):
    self.net, self.sample = Network(env, seed), sample
    self.replay = rollouts.LaneReplay(env, capacity, seed=seed)
    for x in (self.replay.obs_tm1, self.replay.actions, self.replay.transitions.observation,
              self.replay.transitions.reward, self.replay.transitions.discount):
      x.zero_()                 # as the torch agent's rings start, so whole rings compare
    self.out = self.replay.make_batch(sample)

  def select_policy(self, timestep):
    return rollouts.EpsilonGreedy(self.net(timestep.observation), EPSILON)

  def update(self, timestep, actions, new_timestep):
    self.batch = self.replay.sample(self.sample, out=self.out)


def same_rings(torch_agent, record_agent):
  r = record_agent.replay
  env = torch_agent.env
  if not torch.equal(torch_agent.num_added, r.num_added):
    return False
  parts_tm1 = env.split_observation(r.obs_tm1) if env.ragged else (r.obs_tm1,)
  parts = env.split_observation(r.transitions.observation) if env.ragged else (r.transitions.observation,)
  pairs = list(zip(torch_agent.obs_tm1, parts_tm1)) + list(zip(torch_agent.obs, parts)) + [
      (torch_agent.actions, r.actions), (torch_agent.reward, r.transitions.reward),
      (torch_agent.discount, r.transitions.discount)]
  return all(torch.equal(a, b) for a, b in pairs)


def wall(fn):
  torch.cuda.synchronize()
  t0 = time.perf_counter()
  out = fn()
  torch.cuda.synchronize()
  return time.perf_counter() - t0, out


def capacity_for(env, ring_bytes):
  row = max(int(p[0].numel()) for p in env.split_observation(env.make_buffers().observation)) * 4
  cap = 10000
  while cap > 1 and cap * env.batch * (2 * row + 16) > ring_bytes:
    cap //= 2
  return cap


def sample_kernel(agent, size, reps=20):
  """(µs per sample, achieved bytes/s) of LaneReplay.sample on the filled rings, timed with CUDA events."""
  r = agent.replay
  env = r.environment
  out = r.make_batch(size)
  for _ in range(3):
    r.sample(size, out=out)
  start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  start.record()
  for _ in range(reps):
    r.sample(size, out=out)
  end.record()
  torch.cuda.synchronize()
  seconds = start.elapsed_time(end) / 1e3 / reps
  ready = r.size >= 1
  rows = sum(int(p[0].numel()) * p.element_size() for p in env.split_observation(r.transitions.observation[0])) \
      if env.ragged else int(r.transitions.observation[0].numel()) * r.transitions.observation.element_size()
  per_transition = 2 * rows / env.batch + 4 + r.transitions.reward.element_size() + 4      # o_tm1, o_t, a, r, d
  moved = 2 * per_transition * size * int(ready.sum()) + 9 * env.batch                   # read + write; counts, ready
  return seconds * 1e6, moved / seconds


def one_environment(bsuite_id, B, episodes, rounds, sample, ring_bytes):
  times = {'torch': [], 'record': []}
  equal, calls, kernel = True, {}, None
  for r in range(rounds):
    for kind in (('torch', 'record') if r % 2 == 0 else ('record', 'torch')):
      env = bsuite_b200.load_from_id(bsuite_id, batch=B, device='cuda', seed=1 + r)
      cap = capacity_for(env, ring_bytes)
      agent = TorchAgent(env, 3, cap, episodes, sample) if kind == 'torch' else RecordAgent(env, 3, cap, sample)
      seconds, n = wall(lambda: rollouts.run_episodes(agent, env, num_episodes=episodes, policy_seed=POLICY_SEED))
      times[kind].append(seconds / n * 1e6)
      calls[kind] = n
      if kind == 'torch':
        torch_agent = agent
      else:
        record_agent = agent
    equal = equal and same_rings(torch_agent, record_agent)
    if r == rounds - 1:
      kernel = sample_kernel(record_agent, sample)
    del torch_agent, record_agent
  t, rec = statistics.median(times['torch']), statistics.median(times['record'])
  print(json.dumps(dict(case='run_episodes', bsuite_id=bsuite_id, batch=B, capacity=cap, episodes=episodes,
                        sample=sample, torch_us_per_call=round(t, 1), record_us_per_call=round(rec, 1),
                        speedup=round(t / rec, 2), calls=calls, rings_bit_equal=equal,
                        sample_kernel_us=round(kernel[0], 2), sample_kernel_GBps=round(kernel[1] / 1e9, 1),
                        fraction_of_3_35_TBps=round(kernel[1] / HBM, 3))), flush=True)


def whole_sweep(lanes, capacity, episodes, rounds, sample):
  times = {'torch': [], 'record': []}
  equal = True
  for r in range(rounds):
    for kind in (('torch', 'record') if r % 2 == 0 else ('record', 'torch')):
      batch = suite.SweepBatch(sweep.SWEEP, lanes=lanes, device='cuda', seed=2 + r, packed=True)
      if kind == 'torch':
        agents = {k: TorchAgent(env, i, capacity, episodes, sample) for i, (k, env) in enumerate(batch.envs.items())}
      else:
        agents = {k: RecordAgent(env, i, capacity, sample) for i, (k, env) in enumerate(batch.envs.items())}
      seconds, calls = wall(lambda: batch.run_episodes(agents, num_episodes=episodes, policy_seed=POLICY_SEED))
      times[kind].append(seconds / max(calls.values()) * 1e6)
      if kind == 'torch':
        torch_agents = agents
      else:
        record_agents = agents
      batch.close()
    equal = equal and all(same_rings(torch_agents[k], record_agents[k]) for k in torch_agents)
  t, rec = statistics.median(times['torch']), statistics.median(times['record'])
  print(json.dumps(dict(case='sweep', packs=len(torch_agents), lanes=lanes, capacity=capacity, episodes=episodes,
                        sample=sample, torch_us_per_lock_step=round(t, 1), record_us_per_lock_step=round(rec, 1),
                        speedup=round(t / rec, 2), rings_bit_equal=equal)), flush=True)


def main():
  p = argparse.ArgumentParser()
  p.add_argument('--batches', type=int, nargs='+', default=[64, 1024, 4096])
  p.add_argument('--ids', nargs='+', default=['catch/0', 'deep_sea/0', 'cartpole/0'])
  p.add_argument('--episodes', type=int, default=3)
  p.add_argument('--rounds', type=int, default=3)
  p.add_argument('--sample', type=int, default=32)
  p.add_argument('--ring-bytes', type=float, default=2e9)
  p.add_argument('--lanes', type=int, default=64)
  p.add_argument('--sweep-capacity', type=int, default=16)
  p.add_argument('--sweep-episodes', type=int, default=2)
  p.add_argument('--sweep-rounds', type=int, default=1)
  args = p.parse_args()
  with tempfile.TemporaryDirectory() as tmp:
    os.environ[datasets.ENV_VAR] = datasets.write_synthetic_mnist(tmp, 4096, 16, 0)
    for bsuite_id in args.ids:
      for B in args.batches:
        one_environment(bsuite_id, B, args.episodes, args.rounds, args.sample, args.ring_bytes)
    if args.lanes > 0:
      whole_sweep(args.lanes, args.sweep_capacity, args.sweep_episodes, args.sweep_rounds, args.sample)
  print(json.dumps(dict(card=card())), flush=True)


if __name__ == '__main__':
  main()
