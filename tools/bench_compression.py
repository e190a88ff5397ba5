#!/usr/bin/env python
"""A/B of observation buffers in plain device memory against the compressible pool (bsuite_b200/obs_memory.py).

    python tools/bench_compression.py [--out out/compression.jsonl] [--only deep_sea,catch] [--rounds 3]

Prints the card, its power limit, the generic-compression attribute and what bsb_obs_memory_info counts, then for
each row times, per arm (plain `torch.empty` observations, pool observations) and alternating the arms each round:
  step    : single-step launches cycling through a ring of output buffers larger than the L2
  graph   : G single-step launches replayed from one CUDA graph (each writing its own buffer set)
  rollout : one launch of T = 16 fused steps
Both arms step twin environments (same seed, same actions, same calls), so their outputs must be bit-equal; the
tool checks that after the last round and exits non-zero if not.  Row selection in obs_memory.COMPRESSED_FAMILIES
rests on these numbers: a family is kept on plain memory when its pool arm is slower beyond the plain arm's range.
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
from bsuite_b200 import datasets, obs_memory  # noqa: E402

# name, bsuite_id, batch, obs_dtype
ROWS = [
    ('deep_sea/11 N=32', 'deep_sea/11', 65536, 'float32'),
    ('deep_sea/11 N=32 bf16', 'deep_sea/11', 65536, 'bfloat16'),
    ('deep_sea/11 N=32 uint8', 'deep_sea/11', 65536, 'uint8'),
    ('deep_sea/0 N=10', 'deep_sea/0', 262144, 'float32'),
    ('catch/0', 'catch/0', 131072, 'float32'),
    ('mnist/0', 'mnist/0', 65536, 'float32'),
    ('cartpole/0', 'cartpole/0', 131072, 'float32'),
    ('mountain_car/0', 'mountain_car/0', 131072, 'float32'),
    ('bandit/0', 'bandit/0', 1048576, 'float32'),
    ('umbrella_distract/22', 'umbrella_distract/22', 65536, 'float32'),
]
ROLLOUT_T = 16


def events_time(fn, n):
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  e0.record()
  for i in range(n):
    fn(i)
  e1.record()
  torch.cuda.synchronize()
  return e0.elapsed_time(e1) * 1e-3 / n


class Arm:
  """One environment and its output buffers, all observations from `pool` (None: torch's default allocator)."""

  def __init__(self, bsuite_id, batch, obs_dtype, pool, ring_n, graph_n):
    self.env = bsuite_b200.load_from_id(bsuite_id, batch=batch, device='cuda', seed=0, obs_dtype=obs_dtype)
    self.pool = pool
    self.ring = [self.buffers(None) for _ in range(ring_n)]
    self.roll = self.buffers(ROLLOUT_T)
    self.gbufs = [self.buffers(None) for _ in range(graph_n)]
    self.graph = None

  def buffers(self, num_steps):
    out = self.env.make_buffers(num_steps)
    shape, dtype = out.observation.shape, out.observation.dtype
    if self.pool is None:
      out.observation = torch.empty(shape, dtype=dtype, device='cuda')
    else:
      with torch.cuda.use_mem_pool(self.pool):
        out.observation = torch.empty(shape, dtype=dtype, device='cuda')
    return out

  def capture(self, acts):
    self.env.step(acts[0], out=self.gbufs[0])
    torch.cuda.synchronize()
    self.graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(self.graph, capture_error_mode='thread_local'):
      for g, out in enumerate(self.gbufs):
        self.env.step(acts[g], out=out)

  def outputs(self):
    """Every output tensor this arm wrote, as host arrays."""
    got = []
    for out in self.ring + [self.roll] + self.gbufs:
      got += [out.observation.view(torch.uint8).cpu(), out.reward.cpu(), out.discount.cpu(), out.step_type.cpu()]
    return got


def run_row(name, bsuite_id, batch, obs_dtype, pool, rounds, steps):
  elem = {'float32': 4, 'bfloat16': 2, 'uint8': 1}[obs_dtype]
  probe = bsuite_b200.load_from_id(bsuite_id, batch=1, device='cuda', seed=0)
  numel = 1
  for d in probe.obs_shape:
    numel *= d
  probe.close()
  obs_bytes = batch * numel * elem
  ring_n = max(2, min(8, int(300e6 // max(obs_bytes, 1)) + 1))
  graph_n = ring_n
  acts = torch.randint(0, 3, (steps + graph_n, batch), device='cuda', dtype=torch.int32)
  arms = {'plain': Arm(bsuite_id, batch, obs_dtype, None, ring_n, graph_n),
          'pool': Arm(bsuite_id, batch, obs_dtype, pool, ring_n, graph_n)}
  for arm in arms.values():
    acts.remainder_(arm.env.num_actions)
    for i in range(2 * ring_n):                    # warm-up: module load, every buffer touched once
      arm.env.step(acts[i], out=arm.ring[i % ring_n])
    arm.env.rollout(ROLLOUT_T, out=arm.roll)
    arm.capture(acts)
  torch.cuda.synchronize()
  times = {a: {'step': [], 'graph': [], 'rollout': []} for a in arms}
  for _ in range(rounds):
    for a, arm in arms.items():
      times[a]['step'].append(events_time(lambda i, arm=arm: arm.env.step(acts[i], out=arm.ring[i % ring_n]), steps))
      times[a]['graph'].append(events_time(lambda i, arm=arm: arm.graph.replay(), max(4, steps // graph_n)) / graph_n)
      times[a]['rollout'].append(events_time(lambda i, arm=arm: arm.env.rollout(ROLLOUT_T, out=arm.roll), 6) / ROLLOUT_T)
  equal = all(torch.equal(x, y) for x, y in zip(arms['plain'].outputs(), arms['pool'].outputs()))
  row = dict(name=name, bsuite_id=bsuite_id, batch=batch, obs_dtype=obs_dtype, obs_bytes=obs_bytes, bit_equal=equal)
  line = f'{name:24s} B={batch:8d}'
  for leg in ('step', 'graph', 'rollout'):
    p, q = sorted(times['plain'][leg]), sorted(times['pool'][leg])
    row[leg] = {'plain_us': [t * 1e6 for t in p], 'pool_us': [t * 1e6 for t in q]}
    line += (f' | {leg} plain {p[0] * 1e6:7.1f}-{p[-1] * 1e6:7.1f} pool {q[0] * 1e6:7.1f}-{q[-1] * 1e6:7.1f} us'
             f' x{p[len(p) // 2] / q[len(q) // 2]:.2f}')
  print(line + ('' if equal else '  OUTPUTS DIFFER'), flush=True)
  for arm in arms.values():
    arm.graph = None
    arm.env.close()
  return row


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--out', default=None)
  ap.add_argument('--only', default=None)
  ap.add_argument('--rounds', type=int, default=3)
  ap.add_argument('--steps', type=int, default=80)
  args = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit('bench_compression needs a CUDA device')
  smi = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader', '-i', '0'],
                       capture_output=True, text=True).stdout.strip()
  print(f'card: {torch.cuda.get_device_name(0)} | nvidia-smi: {smi}')
  pool = obs_memory.pool(0)
  supported, compressed, plain = obs_memory.info(0)
  print(f'generic compression attribute: {int(supported)}; pool: {"created" if pool is not None else "none"}')
  if pool is None:
    raise SystemExit('no compressible pool on this device: nothing to compare')
  mnist_dir = '/tmp/bsb_bench_mnist'
  datasets.write_synthetic_mnist(mnist_dir, 4096, 16, 0)
  os.environ[datasets.ENV_VAR] = mnist_dir
  rows, all_equal = [], True
  for name, bsuite_id, batch, obs_dtype in ROWS:
    if args.only and not any(o in name for o in args.only.split(',')):
      continue
    row = run_row(name, bsuite_id, batch, obs_dtype, pool, args.rounds, args.steps)
    supported, compressed, plain = obs_memory.info(0)
    row.update(compressed_bytes_live=compressed, plain_bytes_live=plain)
    print(f'{"":24s} bsb_obs_memory_info while the row ran: compressed {compressed / 1e6:.1f} MB, plain {plain / 1e6:.1f} MB',
          flush=True)
    all_equal &= row['bit_equal']
    rows.append(row)
    torch.cuda.empty_cache()
  if args.out:
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, 'w') as fh:
      for r in rows:
        fh.write(json.dumps(r) + '\n')
  if not all_equal:
    raise SystemExit('pool and plain outputs differ')


if __name__ == '__main__':
  main()
