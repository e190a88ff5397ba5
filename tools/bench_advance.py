#!/usr/bin/env python
"""Output-free masked rollouts (`advance`, bsb_advance_masked) against output-writing masked rollouts, on one GPU.

    python tools/bench_advance.py [--batch 65536] [--lanes 1024] [--steps-per-launch 64 512] [--compare-max-size 12]

(a) One id per experiment at `batch` lanes: lane-steps per second of `advance(64)` and of `rollout(64, mask=full)`
    (every lane active, no budgets), timed in alternation with CUDA events around `iters` calls after a warm-up,
    `rounds` times each; medians are reported, with the observation bytes the rollout writes per launch.
(b) The packed 468-id sweep (`SweepBatch(lanes=L, packed=True, record_rows=True)`) to every id's real episode budget
    through `SweepBatch.run_random_episodes`, once per `--steps-per-launch`: wall time from the first reset to a
    synchronise after the last launch, and the lane-steps played (the steps column of the per-setting sums).  Then
    the same sweep driven pack by pack with output-writing masked rollouts of 64 calls (`rollout(64, out=...,
    mask=..., episodes_left=...)`), timed the same way and compared with the advanced sweep bit for bit (per-setting
    sums, every id's log rows, bsuite scores).  deep_sea's output-writing rollouts write 10^4 * N^3 * 4 bytes per
    lane at the real budget (34 GB per lane over all 21 sizes), so the comparison keeps deep_sea and
    deep_sea_stochastic sizes up to `--compare-max-size` and times both paths on that sweep.

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

import torch  # noqa: E402

import bsuite_b200  # noqa: E402
from bsuite_b200 import analysis, datasets, rollouts, suite, sweep  # noqa: E402


def card():
  try:
    out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                         capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
  except (OSError, subprocess.SubprocessError, IndexError):
    out = 'nvidia-smi unavailable'
  return dict(torch_name=torch.cuda.get_device_name(), nvidia_smi=out)


def timed(fn, iters):
  torch.cuda.synchronize()
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  e0.record()
  for _ in range(iters):
    fn()
  e1.record()
  torch.cuda.synchronize()
  return e0.elapsed_time(e1) / iters


def alternate(fns, iters, rounds):
  samples = {k: [] for k in fns}
  for _ in range(rounds):
    for k, fn in fns.items():
      samples[k].append(timed(fn, iters))
  return {k: statistics.median(v) for k, v in samples.items()}


def per_experiment(batch, T, iters, rounds):
  for bsuite_id in suite.one_per_experiment():
    env = bsuite_b200.load_from_id(bsuite_id, batch=batch, device='cuda', seed=0, track_episodes=True)
    mask = torch.ones(batch, dtype=torch.bool, device='cuda')
    out = env.make_buffers(T)
    env.reset(out=env.make_buffers(), mask=mask)
    fns = dict(advance=lambda: env.advance(T, mask=mask),
               rollout=lambda: env.rollout(T, out=out, mask=mask))
    for fn in fns.values():
      fn()
    ms = alternate(fns, iters, rounds)
    rate = {k: batch * T / (v * 1e-3) for k, v in ms.items()}
    print(json.dumps(dict(part='a', bsuite_id=bsuite_id, batch=batch, T=T, ms_per_launch=ms, lane_steps_per_s=rate,
                          speedup=ms['rollout'] / ms['advance'],
                          rollout_obs_bytes_per_launch=out.observation.numel() * out.observation.element_size())),
          flush=True)
    env.close()
    del out
    torch.cuda.empty_cache()


def driven(batch, T):
  """The sweep driven pack by pack with output-writing masked rollouts of T calls (each pack to its budgets)."""
  for env in batch.envs.values():
    left = rollouts.episode_budget(env)
    mask = left > 0
    env.reset(out=env.make_buffers(), mask=mask)
    out = env.make_buffers(T)
    while bool((left > 0).any()):
      env.rollout(T, out=out, mask=mask, episodes_left=left)


def wall(fn):
  torch.cuda.synchronize()
  start = time.perf_counter()
  result = fn()
  torch.cuda.synchronize()
  return time.perf_counter() - start, result


def sweep_row(batch, seconds, calls, **extra):
  steps = batch.local_returns()[:, 2].sum().item()
  return dict(part='b', ids=len(batch.bsuite_ids), lanes=batch.lanes, seconds=seconds, lane_steps=steps,
              lane_steps_per_s=steps / seconds, max_calls=max(calls.values()) if calls else None, **extra)


def same_results(a, b):
  if not torch.equal(a.local_returns(), b.local_returns()):
    return False
  rows = {k: (a.envs[k].logged_rows(), b.envs[k].logged_rows()) for k in a.envs}
  for k, (x, y) in rows.items():
    if not (torch.equal(x['counts'], y['counts']) and torch.equal(x['rows'], y['rows'])):
      return False
  sa, sb = analysis.bsuite_score(a), analysis.bsuite_score(b)
  return torch.equal(sa.score.view(torch.int64), sb.score.view(torch.int64)) and torch.equal(sa.finished, sb.finished)


def whole_sweep(lanes, steps_per_launch, compare_max_size, compare=True):
  kw = dict(lanes=lanes, device='cuda', seed=0, record_rows=True, packed=True)
  for T in steps_per_launch:
    batch = suite.SweepBatch(list(sweep.SWEEP), **kw)
    seconds, calls = wall(lambda: batch.run_random_episodes(steps_per_launch=T))
    print(json.dumps(sweep_row(batch, seconds, calls, path='advance', steps_per_launch=T)), flush=True)
    batch.close()
    del batch
    torch.cuda.empty_cache()
  if not compare:
    return
  ids = [i for i in sweep.SWEEP if not i.startswith('deep_sea') or sweep.SETTINGS[i]['size'] <= compare_max_size]
  advanced = suite.SweepBatch(ids, **kw)
  seconds, calls = wall(lambda: advanced.run_random_episodes(steps_per_launch=64))
  print(json.dumps(sweep_row(advanced, seconds, calls, path='advance', steps_per_launch=64,
                             deep_sea_max_size=compare_max_size)), flush=True)
  written = suite.SweepBatch(ids, **kw)
  seconds, _ = wall(lambda: driven(written, 64))
  print(json.dumps(sweep_row(written, seconds, {}, path='rollout', steps_per_launch=64,
                             deep_sea_max_size=compare_max_size, bit_equal=same_results(advanced, written))),
        flush=True)


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--batch', type=int, default=65536)
  ap.add_argument('--T', type=int, default=64)
  ap.add_argument('--iters', type=int, default=10)
  ap.add_argument('--rounds', type=int, default=5)
  ap.add_argument('--lanes', type=int, default=1024)
  ap.add_argument('--steps-per-launch', type=int, nargs='+', default=[64, 512])
  ap.add_argument('--compare-max-size', type=int, default=12)
  ap.add_argument('--skip', choices=['a', 'b', 'compare'], default=None,
                  help='leave out (a), (b), or the output-writing comparison of (b)')
  args = ap.parse_args()
  if not torch.cuda.is_available():
    raise RuntimeError('bench_advance.py measures on a CUDA device; none is available')
  print(json.dumps(dict(card=card())), flush=True)
  with tempfile.TemporaryDirectory() as tmp:
    os.environ[datasets.ENV_VAR] = datasets.write_synthetic_mnist(tmp, 4096, 16, 0)
    if args.skip != 'a':
      per_experiment(args.batch, args.T, args.iters, args.rounds)
    if args.skip != 'b':  # 'compare' runs (b) without the output-writing sweep
      whole_sweep(args.lanes, args.steps_per_launch, args.compare_max_size, compare=args.skip != 'compare')
  print(json.dumps(dict(card=card(), peak_mem_gb=torch.cuda.max_memory_allocated() / 1e9)), flush=True)


if __name__ == '__main__':
  main()
