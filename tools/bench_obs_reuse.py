#!/usr/bin/env python
"""What a deep_sea step costs when its destination already holds an observation, and when it holds anything else.

    python tools/bench_obs_reuse.py [--out out/obs_reuse.json] [--rounds 5] [--parts reads,step,gaps,worst]

Prints the card, its power limit and the generic-compression attribute, then (B = 65 536 lanes of deep_sea/11, float32
observations, 268 MB per step):
  reads : the algorithmic rate of torch's `sum()` and `fill_(0)` over 268 MB buffers in three states: compressible
          pool memory holding zeros, pool memory holding observations written by `env.step`, plain `torch.empty`
          memory holding the same observations.  `sum()` runs over a ring of 4 buffers; every `fill_(0)` of an
          observation buffer is timed on its own, after an untimed step has written the observation back.
  step  : single steps into a ring of 4 pool buffer sets, as bench.py's `value` runs them (CUDA events over the
          whole run), and a 16-step fused rollout.
  gaps  : the same single steps, each between its own pair of events: back to back, and with 100 µs of device idle
          time before each step.
  worst : single steps into pool buffers that were just filled with data that is not an observation (random bits,
          all 1.0), each step timed on its own after an untimed refill, against the same per-step timing into
          buffers that hold the previous observation.
Rounds alternate the legs; each leg reports its median and range over the rounds.
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
from bsuite_b200 import obs_memory  # noqa: E402

BSUITE_ID = 'deep_sea/11'
BATCH = 65536
RING = 4
ROLLOUT_T = 16


def events(fn, n):
  """Seconds per call of fn(i), i = 0 .. n - 1, from CUDA events around all n calls."""
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  e0.record()
  for i in range(n):
    fn(i)
  e1.record()
  torch.cuda.synchronize()
  return e0.elapsed_time(e1) * 1e-3 / n


def each(prepare, fn, n):
  """Median seconds of fn(i) timed on its own, prepare(i) (untimed) before each call."""
  times = []
  for i in range(n):
    prepare(i)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn(i)
    e1.record()
    torch.cuda.synchronize()
    times.append(e0.elapsed_time(e1) * 1e-3)
  return statistics.median(times)


def pool_empty(pool, shape, dtype):
  with torch.cuda.use_mem_pool(pool):
    return torch.empty(shape, dtype=dtype, device='cuda')


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--out', default=None)
  ap.add_argument('--rounds', type=int, default=5)
  ap.add_argument('--steps', type=int, default=200)
  ap.add_argument('--parts', default='reads,step,gaps,worst')
  args = ap.parse_args()
  parts = set(args.parts.split(','))
  if not torch.cuda.is_available():
    raise SystemExit('bench_obs_reuse needs a CUDA device')
  smi = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader', '-i', '0'],
                       capture_output=True, text=True).stdout.strip()
  print(f'card: {torch.cuda.get_device_name(0)} | nvidia-smi: {smi}', flush=True)
  pool = obs_memory.pool(0)
  print(f'generic compression attribute: {int(obs_memory.info(0)[0])}; pool: {"created" if pool is not None else "none"}')
  if pool is None:
    raise SystemExit('no compressible pool on this device')

  env = bsuite_b200.load_from_id(BSUITE_ID, batch=BATCH, device='cuda', seed=0)
  ring = [env.make_buffers() for _ in range(RING)]
  shape, dtype = ring[0].observation.shape, ring[0].observation.dtype
  nbytes = ring[0].observation.numel() * ring[0].observation.element_size()
  acts = torch.randint(0, env.num_actions, (args.steps + 2 * RING, BATCH), device='cuda', dtype=torch.int32)
  for i in range(2 * RING):
    env.step(acts[i], out=ring[i % RING])
  roll = env.make_buffers(ROLLOUT_T)
  env.rollout(ROLLOUT_T, out=roll)
  torch.cuda.synchronize()

  results = {}
  legs = []
  if 'reads' in parts:
    pool_zero = [pool_empty(pool, shape, dtype).zero_() for _ in range(RING)]
    pool_obs = [env.make_buffers() for _ in range(RING)]
    plain_obs = [env.make_buffers() for _ in range(RING)]
    for b in plain_obs:
      b.observation = torch.empty(shape, dtype=dtype, device='cuda')
    for bufs in (pool_obs, plain_obs):
      for i, b in enumerate(bufs):
        env.step(acts[i], out=b)
    states = {'pool zeros': (pool_zero, None), 'pool observations': (pool_obs, True),
              'plain observations': (plain_obs, True)}
    for state, (bufs, is_obs) in states.items():
      tensors = [b if isinstance(b, torch.Tensor) else b.observation for b in bufs]
      legs.append((f'sum   {state}', lambda ts=tensors: events(lambda i: ts[i % RING].sum(), 40)))
      if is_obs:
        legs.append((f'fill0 {state}', lambda bs=bufs: each(lambda i: env.step(acts[i % RING], out=bs[i % RING]),
                                                             lambda i: bs[i % RING].observation.fill_(0), 12)))
      else:
        legs.append((f'fill0 {state}', lambda ts=tensors: events(lambda i: ts[i % RING].fill_(0), 40)))
  if 'step' in parts:
    legs.append(('step  ring of 4 pool buffers', lambda: events(lambda i: env.step(acts[i], out=ring[i % RING]), args.steps)))
    legs.append((f'fused rollout (T = {ROLLOUT_T}, per step)',
                 lambda: events(lambda i: env.rollout(ROLLOUT_T, out=roll), 6) / ROLLOUT_T))
  if 'gaps' in parts:
    def per_step(gap_cycles):
      def run():
        pairs = []
        for i in range(48):
          if gap_cycles:
            torch.cuda._sleep(gap_cycles)
          e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
          e0.record()
          env.step(acts[i], out=ring[i % RING])
          e1.record()
          pairs.append((e0, e1))
        torch.cuda.synchronize()
        return statistics.median(a.elapsed_time(b) for a, b in pairs) * 1e-3
      return run
    legs.append(('step  ring, each timed, back to back', per_step(0)))
    legs.append(('step  ring, each timed, 100 us idle before', per_step(200000)))
  if 'worst' in parts:
    junk = pool_empty(pool, shape, dtype)
    junk.view(torch.int32).random_()                   # random bits: NaN payloads, -0.0, denormals
    ones = pool_empty(pool, shape, dtype).fill_(1.0)
    wbufs = [env.make_buffers() for _ in range(RING)]
    for i, b in enumerate(wbufs):
      env.step(acts[i], out=b)
    legs.append(('step  each, ring, into the previous observation',
                 lambda: each(lambda i: None, lambda i: env.step(acts[i], out=ring[i % RING]), 24)))
    legs.append(('step  each, into the previous observation',
                 lambda: each(lambda i: None, lambda i: env.step(acts[i], out=wbufs[i % RING]), 24)))
    legs.append(('step  each, into random bits',
                 lambda: each(lambda i: wbufs[i % RING].observation.copy_(junk),
                              lambda i: env.step(acts[i], out=wbufs[i % RING]), 24)))
    legs.append(('step  each, into all 1.0',
                 lambda: each(lambda i: wbufs[i % RING].observation.copy_(ones),
                              lambda i: env.step(acts[i], out=wbufs[i % RING]), 24)))

  for _ in range(args.rounds):
    for name, leg in legs:
      results.setdefault(name, []).append(leg())
  summary = {}
  for name, _ in legs:
    t = sorted(results[name])
    med = statistics.median(t)
    summary[name] = {'us': [x * 1e6 for x in t], 'median_us': med * 1e6, 'algorithmic_tbs': nbytes / med / 1e12}
    print(f'{name:44s} {med * 1e6:8.1f} us  ({t[0] * 1e6:.1f}-{t[-1] * 1e6:.1f})  {nbytes / med / 1e12:5.2f} TB/s of 268 MB'
          f'  rounds: {" ".join(f"{x * 1e6:.1f}" for x in results[name])}', flush=True)
  if args.out:
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, 'w') as fh:
      json.dump({'card': torch.cuda.get_device_name(0), 'nvidia_smi': smi, 'legs': summary}, fh, indent=1)
  env.close()


if __name__ == '__main__':
  main()
