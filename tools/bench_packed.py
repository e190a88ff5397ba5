#!/usr/bin/env python
"""One packed handle per experiment against one handle per setting: graph-captured rollouts on one GPU.

    python tools/bench_packed.py [--out out/packed.jsonl] [--lanes 4096] [--only catch,mnist] [--replays 20]

For every experiment whose settings share an observation shape (19 of 23), with `--lanes` lanes per setting:
  separate : one handle per setting, each rollout on a stream of its own (as SuiteBatch / SweepBatch run them)
  packed   : one handle of all settings (bsuite_b200.load_experiment), the same lanes
both captured into one CUDA graph per variant and replayed; T = 1 and T = 64 steps per rollout, actions sampled on
the device.  Then all 19 experiments at T = 1: 386 handles against 19.  Reported per row: µs per replay (median
of `--repeats` windows, alternating the two variants, with the range), env-steps/s, and the kernel launches of one
replay (counted by the library over an eager pass).  The card's name and power limit are printed first.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import bsuite_b200  # noqa: E402
from bsuite_b200 import _lib  # noqa: E402
from bsuite_b200 import sweep  # noqa: E402

SHAPE_CHANGING = ('deep_sea', 'deep_sea_stochastic', 'memory_size', 'umbrella_distract')
PACKABLE = tuple(name for name in sweep.BY_EXPERIMENT if name not in SHAPE_CHANGING)


class Captured:
  """`envs` each running a T-step rollout (sampled actions) on a stream of its own, in one CUDA graph."""

  def __init__(self, envs, T):
    self.envs, self.T = envs, T
    self.outs = [env.make_buffers(T, with_actions=True) for env in envs]
    self.streams = [torch.cuda.Stream() for _ in envs]
    lib = _lib.load()
    before = lib.bsb_launch_count()
    self.record()                         # eager pass: modules load, function attributes are set
    torch.cuda.synchronize()
    self.launches = lib.bsb_launch_count() - before
    self.graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(self.graph, capture_error_mode='thread_local'):
      self.record()
    self.graph.replay()
    torch.cuda.synchronize()

  def record(self):
    cur = torch.cuda.current_stream()
    for env, out, stream in zip(self.envs, self.outs, self.streams):
      stream.wait_stream(cur)
      with torch.cuda.stream(stream):
        env.rollout(self.T, out=out)
    for stream in self.streams:
      cur.wait_stream(stream)

  def time(self, replays):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(replays):
      self.graph.replay()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e-3 / replays


def compare(label, separate_envs, packed_envs, lanes_total, T, args):
  variants = dict(separate=Captured(separate_envs, T), packed=Captured(packed_envs, T))
  times = {k: [] for k in variants}
  for _ in range(args.repeats):             # alternate the two variants
    for k, v in variants.items():
      times[k].append(v.time(args.replays))
  rows = []
  for k, v in variants.items():
    ts = sorted(times[k])
    dt = ts[len(ts) // 2]
    rows.append(dict(config=label, variant=k, T=T, handles=len(v.envs), lanes=lanes_total,
                     launches_per_replay=v.launches, us_per_replay=dt * 1e6, us_range=[ts[0] * 1e6, ts[-1] * 1e6],
                     env_steps_per_s=T * lanes_total / dt))
  del variants
  return rows


def main():
  parser = argparse.ArgumentParser()
  parser.add_argument('--out', default=None)
  parser.add_argument('--lanes', type=int, default=4096)
  parser.add_argument('--only', default='')
  parser.add_argument('--replays', type=int, default=20)
  parser.add_argument('--repeats', type=int, default=3, help='timed windows per variant (median reported)')
  parser.add_argument('--skip-all', action='store_true')
  args = parser.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit('bench_packed.py needs a CUDA device')
  from bsuite_b200 import datasets
  mnist_dir = os.path.join(os.environ.get('TMPDIR', '/tmp'), 'bsb_bench_mnist')
  datasets.write_synthetic_mnist(mnist_dir, 4096, 16, 0)
  os.environ[datasets.ENV_VAR] = mnist_dir
  card = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                        capture_output=True, text=True).stdout.strip().splitlines()
  print(json.dumps(dict(device=torch.cuda.get_device_name(0), nvidia_smi=card[:1])), flush=True)
  only = [s for s in args.only.split(',') if s]
  rows = []
  L = args.lanes

  def emit(new_rows):
    for row in new_rows:
      rows.append(row)
      print(json.dumps(row), flush=True)

  for name in PACKABLE:
    if only and name not in only:
      continue
    for T in (1, 64):
      pack = bsuite_b200.load_experiment(name, L, device='cuda', seed=0)
      parts = [bsuite_b200.load_from_id(i, batch=L, device='cuda', seed=0) for i in pack.bsuite_ids]
      emit(compare(name, parts, [pack], pack.batch, T, args))
      del pack, parts
      torch.cuda.empty_cache()
  if not args.skip_all and not only:
    packs = [bsuite_b200.load_experiment(name, L, device='cuda', seed=0) for name in PACKABLE]
    parts = [bsuite_b200.load_from_id(i, batch=L, device='cuda', seed=0) for p in packs for i in p.bsuite_ids]
    emit(compare(f'all_{len(PACKABLE)}_experiments', parts, packs, sum(p.batch for p in packs), 1, args))
  if args.out:
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, 'w') as f:
      for row in rows:
        f.write(json.dumps(row) + '\n')


if __name__ == '__main__':
  main()
