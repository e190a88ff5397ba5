#!/usr/bin/env python
"""Per-family throughput table on one GPU: single-step launches and T-fused rollouts.

    python tools/bench_families.py [--out out/families.jsonl] [--only catch,mnist] [--batch 4096] [--graph 16]
                                   [--obs-dtype float32|bfloat16|uint8]

For every configuration: env-steps/s and the algorithmic-bytes bandwidth (SURVEY.md 8d formula:
s*obs_numel + 4 action + 4 reward + 4 discount + 4 step_type + state read/write, s = 4, 2 or 1 bytes per observation
element) for
  step    : K single-step launches, caller-provided device actions, outputs cycling through a ring > L2
  rollout : one launch of T fused steps with on-device Philox actions, [T,B,...] outputs
  cast    : (reduced --obs-dtype only) what a user of a float32 environment does instead: a float32 step followed by
            `observation.to(dtype)`, the same ring of outputs
--obs-dtype uint8 runs the deep_sea and catch rows only (the families whose observations are 0 / 1).
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import bsuite_b200  # noqa: E402
from bsuite_b200 import datasets  # noqa: E402

# name, (kind, spec, kwargs), batch, state bytes (read+write) per lane-step
CONFIGS = [
    ('deep_sea/11 N=32', ('id', 'deep_sea/11', {}), 65536, 8),
    ('deep_sea/0 N=10', ('id', 'deep_sea/0', {}), 262144, 8),
    ('deep_sea/20 N=50', ('id', 'deep_sea/20', {}), 32768, 8),
    ('deep_sea_stochastic/11', ('id', 'deep_sea_stochastic/11', {}), 65536, 8 + 16 + 16),
    ('catch/0', ('id', 'catch/0', {}), 131072, 8 + 16),
    ('catch_noise/0', ('id', 'catch_noise/0', {}), 131072, 8 + 16 + 32),
    ('cartpole/0', ('id', 'cartpole/0', {}), 131072, 2 * (48 + 8 + 4) + 16),
    ('cartpole_swingup/0', ('id', 'cartpole_swingup/0', {}), 131072, 2 * (48 + 8 + 4) + 16),
    ('mountain_car/0', ('id', 'mountain_car/0', {}), 131072, 2 * (16 + 8 + 4) + 16),
    ('memory_len/5', ('id', 'memory_len/5', {}), 262144, 2 * 12 + 16),
    ('memory_size/16 (40 bits)', ('id', 'memory_size/16', {}), 131072, 2 * 12 + 16),
    ('bandit/0', ('id', 'bandit/0', {}), 1048576, 8),
    ('discounting_chain/0', ('id', 'discounting_chain/0', {}), 1048576, 8),
    ('umbrella_length/10 (n=20)', ('id', 'umbrella_length/10', {}), 131072, 8 + 16),
    ('umbrella_distract/22 (n=100)', ('id', 'umbrella_distract/22', {}), 65536, 8 + 16),
    ('mnist/0 (synthetic 4096 imgs)', ('id', 'mnist/0', {}), 65536, 8 + 16),
]


def measure(fn, iters, warm=3):
  for _ in range(warm):
    fn()
  torch.cuda.synchronize()
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  e0.record()
  for i in range(iters):
    fn(i)
  e1.record()
  torch.cuda.synchronize()
  return e0.elapsed_time(e1) * 1e-3 / iters


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--out', default=None)
  ap.add_argument('--only', default=None)
  ap.add_argument('--steps', type=int, default=60)
  ap.add_argument('--rollout', type=int, default=16)
  ap.add_argument('--batch', type=int, default=0, help='override every configuration\'s batch size')
  ap.add_argument('--graph', type=int, default=0, help='also time G single-step launches replayed from one CUDA graph')
  ap.add_argument('--obs-dtype', default='float32', choices=('float32', 'bfloat16', 'uint8'))
  args = ap.parse_args()
  dtype = dict(float32=torch.float32, bfloat16=torch.bfloat16, uint8=torch.uint8)[args.obs_dtype]
  elem = torch.empty((), dtype=dtype).element_size()
  mnist_dir = '/tmp/bsb_bench_mnist'
  datasets.write_synthetic_mnist(mnist_dir, 4096, 16, 0)
  os.environ[datasets.ENV_VAR] = mnist_dir
  rows = []
  for name, (kind, what, kw), batch, state_bytes in CONFIGS:
    if args.only and not any(o in name for o in args.only.split(',')):
      continue
    if args.obs_dtype == 'uint8' and not name.startswith(('deep_sea', 'catch')):
      continue
    if args.batch:
      batch = args.batch
    env = bsuite_b200.load_from_id(what, batch=batch, device='cuda', seed=0, obs_dtype=args.obs_dtype)
    numel = 1
    for d in env.obs_shape:
      numel *= d
    bytes_per = elem * numel + 16 + state_bytes
    obs_bytes = batch * numel * elem
    ring_n = max(2, min(8, int(300e6 // max(batch * numel * 4, 1)) + 1))
    ring = [env.make_buffers() for _ in range(ring_n)]
    acts = torch.randint(0, env.num_actions, (args.steps + 8, batch), device='cuda', dtype=torch.int32)
    step_s = measure(lambda i=0: env.step(acts[i % acts.shape[0]], out=ring[i % ring_n]), args.steps)
    cast_s = None
    if dtype != torch.float32:
      env32 = bsuite_b200.load_from_id(what, batch=batch, device='cuda', seed=0)
      ring32 = [env32.make_buffers() for _ in range(ring_n)]
      cast_s = measure(lambda i=0: env32.step(acts[i % acts.shape[0]], out=ring32[i % ring_n]).observation.to(dtype),
                       args.steps)
      env32.close()
      del ring32
    T = args.rollout
    while T > 1 and T * obs_bytes > 6e9:
      T //= 2
    rbuf = env.make_buffers(T)
    roll_s = measure(lambda i=0: env.rollout(T, out=rbuf), 6, warm=2) / T
    graph_s = None
    if args.graph:
      G = args.graph
      while G > 1 and G * obs_bytes > 3e9:
        G //= 2
      genv = bsuite_b200.load_from_id(what, batch=batch, device='cuda', seed=0, obs_dtype=args.obs_dtype)
      graphed = genv.capture(G)                      # G per-step launches, caller-provided actions
      graphed.actions.copy_(acts[:G])
      graph_s = measure(lambda i=0: graphed.replay(), max(3, args.steps // G), warm=2) / G
      del graphed
      # the same handle stepped EAGERLY afterwards: it stays in graph-safe mode (step counter and chunk scheduler
      # on the device), so this isolates the mode's kernel-side cost from the graph launch mechanics
      gsafe_s = measure(lambda i=0: genv.step(acts[i % acts.shape[0]], out=ring[i % ring_n]), args.steps)
      genv.close()
    row = dict(name=name, batch=batch, obs_numel=numel, bytes_per_lane_step=bytes_per,
               step_us=step_s * 1e6, step_steps_per_s=batch / step_s, step_gbs=batch * bytes_per / step_s / 1e9,
               rollout_T=T, rollout_us_per_step=roll_s * 1e6, rollout_steps_per_s=batch / roll_s,
               rollout_gbs=batch * bytes_per / roll_s / 1e9)
    rows.append(row)
    print(f"{name:32s} B={batch:8d} K={numel:5d}  step {row['step_us']:8.1f} us {row['step_steps_per_s']:.3e}/s "
          f"{row['step_gbs']:7.0f} GB/s | rollout(T={T}) {row['rollout_us_per_step']:8.1f} us/step "
          f"{row['rollout_steps_per_s']:.3e}/s {row['rollout_gbs']:7.0f} GB/s"
          + ('' if graph_s is None else f" | graph {graph_s * 1e6:7.1f} us/step, eager in graph-safe mode {gsafe_s * 1e6:7.1f}"), flush=True)
    if cast_s is not None:
      row.update(obs_dtype=args.obs_dtype, cast_us=cast_s * 1e6, cast_steps_per_s=batch / cast_s)
      print(f"{'':32s} float32 step + .to({args.obs_dtype}): {cast_s * 1e6:8.1f} us {batch / cast_s:.3e}/s", flush=True)
    row['obs_dtype'] = args.obs_dtype
    if graph_s is not None:
      row.update(graph_us_per_step=graph_s * 1e6, graph_steps_per_s=batch / graph_s, graph_safe_eager_us=gsafe_s * 1e6)
    env.close()
    del ring, rbuf, acts
    torch.cuda.empty_cache()
  if args.out:
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, 'w') as fh:
      for r in rows:
        fh.write(json.dumps(r) + '\n')


if __name__ == '__main__':
  main()
