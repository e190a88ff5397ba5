#!/usr/bin/env python
"""Next-step against same-step auto-reset on one GPU: µs per call, transitions per second and algorithmic GB/s.

    python tools/bench_autoreset.py [--out out/autoreset.jsonl] [--only catch,mnist] [--rollout 16] [--iters 50]

For every configuration of tools/bench_families.py (same batch sizes), plus memory_len/0, and both `autoreset` modes:
  step    : single-step launches with caller-provided device actions
  rollout : one launch of `--rollout` fused steps with on-device Philox actions
A transition is a timestep whose step_type is not FIRST, counted on the device over the timed calls themselves (each
call writes its step types to a slice of its own).  `--repeats` windows per mode, the median reported with the range
of µs per call.  Under next-step
a lane spends one call per episode on its reset (FIRST); under same-step that call is merged into the LAST one.
GB/s counts the observation bytes of every call plus the scalars and the state, as bench_families.py does (no
final observations are requested).  Last, the 23-experiment SweepBatch (4 096 lanes each) in both modes: a fused
16-step rollout and its graph replay.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

import torch  # noqa: E402

import bsuite_b200  # noqa: E402
import bench_families as bf  # noqa: E402


def _time(fn, n):
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  e0.record()
  for i in range(n):
    fn(i)
  e1.record()
  torch.cuda.synchronize()
  return e0.elapsed_time(e1) * 1e-3 / n


def run_config(name, spec, batch, state_bytes, autoreset, args):
  """`args.repeats` timed windows per mode; each call of a window writes its step types to a slice of its own, so the
  transitions counted are those of the timed calls themselves.  Reports the median window."""
  from bsuite_b200.environment import StepBuffers
  kind, target, kwargs = spec
  env = bsuite_b200.load_from_id(target, batch=batch, device='cuda', seed=0, autoreset=autoreset, **kwargs)
  obs_bytes = 4 * int(torch.tensor(env.obs_shape).prod())
  per_lane = obs_bytes + 16 + state_bytes
  T, n = args.rollout, args.iters
  ring = [env.make_buffers() for _ in range(4)]             # observations cycle through a ring > L2
  step_types = torch.empty((n, batch), dtype=torch.int32, device='cuda')
  step_out = [StepBuffers(ring[i % 4].observation, ring[i % 4].reward, ring[i % 4].discount, step_types[i])
              for i in range(n)]
  acts = torch.randint(0, env.num_actions, (n, batch), dtype=torch.int32, device='cuda')
  reps = max(3, n // T)
  roll = env.make_buffers(T, with_actions=True)
  roll_types = torch.empty((reps, T, batch), dtype=torch.int32, device='cuda')
  roll_out = [StepBuffers(roll.observation, roll.reward, roll.discount, roll_types[r], roll.actions) for r in range(reps)]
  windows = {'step': [], f'rollout{T}': []}
  for i in range(3):
    env.step(acts[i], out=step_out[i])
  env.rollout(T, out=roll_out[0])
  torch.cuda.synchronize()
  for _ in range(args.repeats):
    dt = _time(lambda i: env.step(acts[i], out=step_out[i]), n)
    windows['step'].append((dt, int((step_types != 0).sum()) / n, batch))
    dt = _time(lambda r: env.rollout(T, action_seed=r, out=roll_out[r]), reps)
    windows[f'rollout{T}'].append((dt, int((roll_types != 0).sum()) / reps, T * batch))
  env.close()
  rows = []
  for mode, ws in windows.items():
    dts = sorted(w[0] for w in ws)
    dt, transitions, steps = sorted(ws)[len(ws) // 2]
    rows.append(dict(config=name, autoreset=autoreset, mode=mode, batch=batch, us_per_call=dt * 1e6,
                     us_range=[dts[0] * 1e6, dts[-1] * 1e6], transitions_per_s=transitions / dt,
                     env_steps_per_s=steps / dt, gbps=steps * per_lane / dt / 1e9, windows=len(ws)))
  return rows


def run_sweep(autoreset, args):
  from bsuite_b200.suite import SweepBatch
  batch = SweepBatch(lanes=4096, device='cuda', seed=0, autoreset=autoreset, track_episodes=False)
  T = 16
  outs = {k: env.make_buffers(T, with_actions=True) for k, env in batch.envs.items()}

  def fused():
    for k, env in batch.envs.items():
      env.rollout(T, out=outs[k])

  fused()
  torch.cuda.synchronize()
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  e0.record()
  for _ in range(10):
    fused()
  e1.record()
  torch.cuda.synchronize()
  dt_fused = e0.elapsed_time(e1) * 1e-3 / 10
  fused_transitions = sum(int((o.step_type != 0).sum()) for o in outs.values())    # of the last timed call
  graph = torch.cuda.CUDAGraph()
  stream = torch.cuda.Stream()
  stream.wait_stream(torch.cuda.current_stream())
  with torch.cuda.stream(stream):
    fused()
  torch.cuda.current_stream().wait_stream(stream)
  torch.cuda.synchronize()
  with torch.cuda.graph(graph, capture_error_mode='thread_local'):
    fused()
  graph.replay()
  torch.cuda.synchronize()
  e0.record()
  for _ in range(10):
    graph.replay()
  e1.record()
  torch.cuda.synchronize()
  dt_graph = e0.elapsed_time(e1) * 1e-3 / 10
  graph_transitions = sum(int((o.step_type != 0).sum()) for o in outs.values())    # of the last replay
  lanes = 4096 * len(batch.envs)
  return [dict(config='sweep_23x4096', autoreset=autoreset, mode=mode, batch=lanes, us_per_call=dt * 1e6,
               transitions_per_s=transitions / dt, env_steps_per_s=T * lanes / dt)
          for mode, dt, transitions in (('fused16', dt_fused, fused_transitions), ('graph16', dt_graph, graph_transitions))]


def main():
  parser = argparse.ArgumentParser()
  parser.add_argument('--out', default=None)
  parser.add_argument('--only', default='')
  parser.add_argument('--rollout', type=int, default=16)
  parser.add_argument('--iters', type=int, default=50)
  parser.add_argument('--repeats', type=int, default=3, help='timed windows per configuration (median reported)')
  parser.add_argument('--skip-sweep', action='store_true')
  args = parser.parse_args()
  from bsuite_b200 import datasets
  mnist_dir = os.path.join(os.environ.get('TMPDIR', '/tmp'), 'bsb_bench_mnist')
  datasets.write_synthetic_mnist(mnist_dir, 4096, 16, 0)
  os.environ[datasets.ENV_VAR] = mnist_dir
  only = [s for s in args.only.split(',') if s]
  rows = []
  print(f'# {torch.cuda.get_device_name(0)}')
  # memory_len/0 (L = 1): three calls per episode under next-step
  configs = bf.CONFIGS + [('memory_len/0 (L=1)', ('id', 'memory_len/0', {}), 262144, 2 * 12 + 16)]
  for name, spec, batch, state_bytes in configs:
    if only and not any(o in name for o in only):
      continue
    for autoreset in ('next_step', 'same_step'):
      for row in run_config(name, spec, batch, state_bytes, autoreset, args):
        rows.append(row)
        print(json.dumps(row), flush=True)
  if not args.skip_sweep:
    for autoreset in ('next_step', 'same_step'):
      for row in run_sweep(autoreset, args):
        rows.append(row)
        print(json.dumps(row), flush=True)
  if args.out:
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, 'w') as f:
      for row in rows:
        f.write(json.dumps(row) + '\n')


if __name__ == '__main__':
  main()
