#!/usr/bin/env python
"""Boot_dqn's per-step machinery on the device -- the ensemble step (`rollouts.EnsembleEpsilonGreedy`,
`bsb_step_budgeted_ensemble`) and bootstrap samples (`LaneReplay(bootstrap=...)`, `bsb_replay_sample_bootstrap`) --
against the same agent keeping its heads, rings, masks and noise in torch.

    python tools/bench_boot_dqn.py [--batches 64 1024 4096] [--episodes 3] [--rounds 2] [--sample 128]
                                   [--min-size 128] [--ring-bytes 2e9] [--lanes 64] [--sweep-capacity 16]

Both agents share one network: the reference boot_dqn default's ensemble of K = 20 MLPs [in, 50, 50, A] plus as many
prior networks (scale 3), fixed random weights, evaluated for all 2K networks with one batched matmul per layer.
Neither does SGD.  Epsilon 0.05 (the default's), one policy seed.
  torch   gathers the active head's rows for `EpsilonGreedy`, redraws the heads of lanes that just ended an episode
          with `torch.randint`, keeps per-lane rings in `update` with torch ops, each transition with its mask ~
          Bernoulli(mask_prob)^K and noise ~ N(0, 1)^K drawn when it is added, and samples `--sample` transitions per
          lane (masks and noise gathered with them) with `torch.randint` and gathers.
  device  passes `EnsembleEpsilonGreedy` (heads kept and redrawn by the step), carries a `LaneReplay` with a
          `Bootstrap`, so every transition is recorded in the step, and samples `--sample` per lane and call with
          `LaneReplay.sample(--sample, --min-size)`, whose launch draws the masks and noise.
The head streams differ (torch's generator against the engine's head stream), so the agents play different episodes:
catch and deep_sea episodes have a fixed length and both agents make the same number of calls; cartpole's need not,
and the report gives both counts and times per call.  Every case runs twice: mask_prob = 1 without noise (the default
agent) and mask_prob = 0.5 with noise.
(a) catch/0, deep_sea/0 and cartpole/0 at each batch size, `--episodes` episodes per lane: wall time per call of
    `rollouts.run_episodes`, the agents alternated `--rounds` times on fresh environments; medians.  Then the bootstrap
    sample kernel alone and `bsb_replay_sample` alone on the same filled rings, timed with CUDA events.
(b) The packed 468-id sweep at `--lanes` lanes per id with `--sweep-capacity` slots: wall time of
    `SweepBatch.run_episodes` per lock-step.  One JSON line per measurement, then one with the card's name and power
    limit.
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

K, PRIOR_SCALE, EPSILON, POLICY_SEED = 20, 3.0, 0.05, 5


def card():
  try:
    out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                         capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
  except (OSError, subprocess.SubprocessError, IndexError):
    out = 'nvidia-smi unavailable'
  return dict(torch_name=torch.cuda.get_device_name(), nvidia_smi=out)


class Ensemble:
  """K MLPs [in, 50, 50, A] and K prior MLPs of the same shape over the zero-padded, flattened observation, as one
  batched matmul per layer over the 2K networks: values [K, B, A] = head + PRIOR_SCALE * prior."""

  def __init__(self, env, seed):
    self.env = env
    g = torch.Generator().manual_seed(seed)
    parts = env.split_observation(env.make_buffers().observation)
    self.size = max(int(p[0].numel()) for p in parts)
    sizes = [self.size, 50, 50, env.num_actions]
    self.layers = [((torch.randn(2 * K, a, b, generator=g) / a ** 0.5).cuda(), torch.zeros(2 * K, 1, b, device='cuda'))
                   for a, b in zip(sizes[:-1], sizes[1:])]

  def __call__(self, observation):
    parts = [p.reshape(p.shape[0], -1).float() for p in self.env.split_observation(observation)]
    x = torch.cat([torch.nn.functional.pad(p, (0, self.size - p.shape[1])) for p in parts])
    x = x.unsqueeze(0).expand(2 * K, -1, -1)
    for k, (w, b) in enumerate(self.layers):
      x = torch.baddbmm(b, x, w)
      if k + 1 < len(self.layers):
        x = torch.relu(x)
    return (x[:K] + PRIOR_SCALE * x[K:]).contiguous()


class TorchAgent:
  """Heads, rings, masks and noise kept in torch."""

  def __init__(self, env, seed, capacity, budget, sample, min_size, mask_prob, noise):
    self.env, self.net, self.capacity, self.sample, self.min_size = env, Ensemble(env, seed), capacity, sample, min_size
    self.mask_prob, self.noise = mask_prob, noise
    B = env.batch
    self.lanes = torch.arange(B, device='cuda')
    self.budget = budget
    self.lasts = torch.zeros(B, dtype=torch.int64, device='cuda')
    self.num_added = torch.zeros(B, dtype=torch.int64, device='cuda')
    self.heads = torch.zeros(B, dtype=torch.int64, device='cuda')
    self.gen = torch.Generator(device='cuda').manual_seed(seed)
    obs = env.make_buffers().observation
    self.parts = env.ragged
    self.obs_tm1 = [torch.zeros((capacity,) + tuple(p.shape), dtype=p.dtype, device='cuda') for p in self._split(obs)]
    self.obs = [torch.zeros_like(x) for x in self.obs_tm1]
    self.actions = torch.zeros((capacity, B), dtype=torch.int32, device='cuda')
    self.reward = torch.zeros((capacity, B), dtype=torch.float32, device='cuda')
    self.discount = torch.zeros((capacity, B), dtype=torch.float32, device='cuda')
    self.masks = torch.zeros((capacity, B, K), dtype=torch.uint8, device='cuda')
    self.noises = torch.zeros((capacity, B, K), dtype=torch.float32, device='cuda') if noise else None
    self.batch = None

  def _split(self, obs):
    return self.env.split_observation(obs) if self.parts else (obs,)

  def select_policy(self, timestep):
    values = self.net(timestep.observation)
    return rollouts.EpsilonGreedy(values[self.heads, self.lanes].contiguous(), EPSILON)

  def update(self, timestep, actions, new_timestep):
    stepped = self.lasts < self.budget
    # a new head where an episode just ended
    ended = (new_timestep.step_type == 2) & (timestep.step_type != 2)
    drawn = torch.randint(0, K, (self.env.batch,), device='cuda', generator=self.gen)
    self.heads = torch.where(ended, drawn, self.heads)
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
    # the transition's bootstrap mask and noise, drawn when it is added (agent.py:171-185)
    mask = (torch.rand((self.env.batch, K), device='cuda', generator=self.gen) < self.mask_prob).to(torch.uint8)
    self.masks[slot, self.lanes] = torch.where(keep.unsqueeze(1), mask, self.masks[slot, self.lanes])
    if self.noises is not None:
      z = torch.randn((self.env.batch, K), device='cuda', generator=self.gen)
      self.noises[slot, self.lanes] = torch.where(keep.unsqueeze(1), z, self.noises[slot, self.lanes])
    self.num_added += keep.to(torch.int64)
    self.lasts += ((new_timestep.step_type == 2) & stepped).to(torch.int64)
    # a minibatch per lane from its filled slots, for the lanes holding min_size (the others' entries are unused)
    n = self.num_added.clamp(1, self.capacity)
    ready = self.num_added >= self.min_size
    idx = torch.randint(0, 1 << 62, (self.sample, self.env.batch), device='cuda', generator=self.gen) % n
    self.batch = [ring[idx, self.lanes] for ring in (self.actions, self.reward, self.discount, self.masks)]
    if self.noises is not None:
      self.batch.append(self.noises[idx, self.lanes])
    for k, (ring_tm1, ring) in enumerate(zip(self.obs_tm1, self.obs)):
      lanes = slice(k * L, (k + 1) * L) if self.parts else slice(None)
      part = idx[:, lanes]
      rows = self.lanes[:ring.shape[1]]
      self.batch += [ring_tm1[part, rows], ring[part, rows]]
    self.batch.append(ready)


class DeviceAgent:
  def __init__(self, env, seed, capacity, sample, min_size, mask_prob, noise):
    self.net, self.sample, self.min_size = Ensemble(env, seed), sample, min_size
    self.heads = torch.zeros(env.batch, dtype=torch.int32, device='cuda')
    self.replay = rollouts.LaneReplay(env, capacity, seed=seed,
                                      bootstrap=rollouts.Bootstrap(K, mask_prob, noise, seed=seed + 1))
    self.out = self.replay.make_batch(sample)

  def select_policy(self, timestep):
    return rollouts.EnsembleEpsilonGreedy(self.net(timestep.observation), self.heads, EPSILON)

  def update(self, timestep, actions, new_timestep):
    self.batch = self.replay.sample(self.sample, min_size=self.min_size, out=self.out)


def wall(fn):
  torch.cuda.synchronize()
  t0 = time.perf_counter()
  out = fn()
  torch.cuda.synchronize()
  return time.perf_counter() - t0, out


def capacity_for(env, ring_bytes):
  row = max(int(p[0].numel()) for p in env.split_observation(env.make_buffers().observation)) * 4
  cap = 10000
  while cap > 1 and cap * env.batch * (2 * row + 16 + 5 * K) > ring_bytes:
    cap //= 2
  return cap


def event_time(fn, reps=20):
  for _ in range(3):
    fn()
  start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  start.record()
  for _ in range(reps):
    fn()
  end.record()
  torch.cuda.synchronize()
  return start.elapsed_time(end) / 1e3 / reps


def sample_kernels(agent, size):
  """(µs per bootstrap sample, µs per plain sample) on the agent's filled rings, timed with CUDA events."""
  r = agent.replay
  plain = rollouts.LaneReplay(r.environment, r.capacity, seed=r.seed)
  for name in ('obs_tm1', 'actions', 'num_added'):
    getattr(plain, name).copy_(getattr(r, name))
  for name in ('observation', 'reward', 'discount', 'step_type'):
    getattr(plain.transitions, name).copy_(getattr(r.transitions, name))
  boot_out, plain_out = r.make_batch(size), plain.make_batch(size)
  boot = event_time(lambda: r.sample(size, out=boot_out))
  base = event_time(lambda: plain.sample(size, out=plain_out))
  return boot * 1e6, base * 1e6


def one_environment(bsuite_id, B, episodes, rounds, sample, min_size, ring_bytes, mask_prob, noise):
  times = {'torch': [], 'device': []}
  calls = {'torch': set(), 'device': set()}
  kernel = None
  for r in range(rounds):
    for kind in (('torch', 'device') if r % 2 == 0 else ('device', 'torch')):
      env = bsuite_b200.load_from_id(bsuite_id, batch=B, device='cuda', seed=1 + r)
      cap = capacity_for(env, ring_bytes)
      m = min(min_size, cap)
      agent = (TorchAgent(env, 3, cap, episodes, sample, m, mask_prob, noise) if kind == 'torch'
               else DeviceAgent(env, 3, cap, sample, m, mask_prob, noise))
      seconds, n = wall(lambda: rollouts.run_episodes(agent, env, num_episodes=episodes, policy_seed=POLICY_SEED))
      times[kind].append(seconds / n * 1e6)
      calls[kind].add(n)
      if kind == 'device' and r == rounds - 1:
        kernel = sample_kernels(agent, sample)
      del agent, env
  t, d = statistics.median(times['torch']), statistics.median(times['device'])
  print(json.dumps(dict(case='run_episodes', bsuite_id=bsuite_id, batch=B, capacity=cap, episodes=episodes,
                        sample=sample, min_size=min(min_size, cap), mask_prob=mask_prob, noise=noise,
                        torch_us_per_call=round(t, 1), device_us_per_call=round(d, 1), speedup=round(t / d, 2),
                        calls={k: sorted(v) for k, v in calls.items()}, same_calls=calls['torch'] == calls['device'],
                        bootstrap_sample_us=round(kernel[0], 2), plain_sample_us=round(kernel[1], 2))), flush=True)


def whole_sweep(lanes, capacity, episodes, rounds, sample, mask_prob, noise):
  times = {'torch': [], 'device': []}
  calls = {}
  m = min(128, capacity)
  for r in range(rounds):
    for kind in (('torch', 'device') if r % 2 == 0 else ('device', 'torch')):
      batch = suite.SweepBatch(sweep.SWEEP, lanes=lanes, device='cuda', seed=2 + r, packed=True)
      if kind == 'torch':
        agents = {k: TorchAgent(env, i, capacity, episodes, sample, m, mask_prob, noise)
                  for i, (k, env) in enumerate(batch.envs.items())}
      else:
        agents = {k: DeviceAgent(env, i, capacity, sample, m, mask_prob, noise)
                  for i, (k, env) in enumerate(batch.envs.items())}
      seconds, c = wall(lambda: batch.run_episodes(agents, num_episodes=episodes, policy_seed=POLICY_SEED))
      times[kind].append(seconds / max(c.values()) * 1e6)
      calls[kind] = max(c.values())
      packs = len(agents)
      del agents
      batch.close()
  t, d = statistics.median(times['torch']), statistics.median(times['device'])
  print(json.dumps(dict(case='sweep', packs=packs, lanes=lanes, capacity=capacity, episodes=episodes, sample=sample,
                        mask_prob=mask_prob, noise=noise, torch_us_per_lock_step=round(t, 1),
                        device_us_per_lock_step=round(d, 1), speedup=round(t / d, 2), lock_steps=calls)), flush=True)


def main():
  p = argparse.ArgumentParser()
  p.add_argument('--batches', type=int, nargs='+', default=[64, 1024, 4096])
  p.add_argument('--ids', nargs='+', default=['catch/0', 'deep_sea/0', 'cartpole/0'])
  p.add_argument('--episodes', type=int, default=3)
  p.add_argument('--rounds', type=int, default=2)
  p.add_argument('--sample', type=int, default=128)
  p.add_argument('--min-size', type=int, default=128)
  p.add_argument('--ring-bytes', type=float, default=2e9)
  p.add_argument('--lanes', type=int, default=64)
  p.add_argument('--sweep-capacity', type=int, default=16)
  p.add_argument('--sweep-episodes', type=int, default=2)
  p.add_argument('--sweep-rounds', type=int, default=1)
  args = p.parse_args()
  with tempfile.TemporaryDirectory() as tmp:
    os.environ[datasets.ENV_VAR] = datasets.write_synthetic_mnist(tmp, 4096, 16, 0)
    for mask_prob, noise in ((1.0, False), (0.5, True)):
      for bsuite_id in args.ids:
        for B in args.batches:
          one_environment(bsuite_id, B, args.episodes, args.rounds, args.sample, args.min_size, args.ring_bytes,
                          mask_prob, noise)
      if args.lanes > 0:
        whole_sweep(args.lanes, args.sweep_capacity, args.sweep_episodes, args.sweep_rounds, args.sample, mask_prob,
                    noise)
  print(json.dumps(dict(card=card())), flush=True)


if __name__ == '__main__':
  main()
