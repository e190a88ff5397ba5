#!/usr/bin/env python
"""deep_sea emitter / launch variants on one GPU, plus a pure-write calibration of the HBM ceiling.

    python tools/bench_variants.py [--out out/variants.jsonl]

The engine reads BSB_BLOCK_THREADS / BSB_DEEP_SEA_BULK / BSB_PDL when a handle is created, so each variant is a
fresh environment in the same process.  Every variant is checked against the first one (bit-exact) on a seeded
action matrix before it is timed.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import bsuite_b200  # noqa: E402


def timeit(fn, iters, warm=5):
  for i in range(warm):
    fn(i)
  torch.cuda.synchronize()
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  e0.record()
  for i in range(iters):
    fn(i)
  e1.record()
  torch.cuda.synchronize()
  return e0.elapsed_time(e1) * 1e-3 / iters


def calibrate_writes(rows):
  """Pure-write kernels over the same 268 MB x 4 ring: what a trivial store stream achieves on this GPU."""
  bufs = [torch.empty(65536 * 1024, dtype=torch.float32, device='cuda') for _ in range(4)]
  for name, fn in (('cudaMemsetAsync (tensor.zero_)', lambda i: bufs[i % 4].zero_()),
                   ('torch fill_(1.0) kernel', lambda i: bufs[i % 4].fill_(1.0))):
    s = timeit(fn, 200)
    gbs = bufs[0].numel() * 4 / s / 1e9
    rows.append(dict(calibration=name, us=s * 1e6, gbs=gbs))
    print(f'calibration {name:34s} {s * 1e6:7.1f} us  {gbs:6.0f} GB/s', flush=True)
  src = torch.empty_like(bufs[0])
  s = timeit(lambda i: bufs[i % 4].copy_(src), 100)
  rows.append(dict(calibration='copy_ (read + write bytes)', us=s * 1e6, gbs=2 * src.numel() * 4 / s / 1e9))
  print(f"calibration {'copy_ (read+write bytes)':34s} {s * 1e6:7.1f} us  {2 * src.numel() * 4 / s / 1e9:6.0f} GB/s", flush=True)


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--out', default=None)
  ap.add_argument('--steps', type=int, default=300)
  args = ap.parse_args()
  rows = []
  calibrate_writes(rows)
  variants = [dict(threads=64, bulk=0, pdl=1, group=0), dict(threads=64, bulk=1, pdl=1, group=0),
              dict(threads=64, bulk=1, pdl=0, group=0), dict(threads=64, bulk=1, pdl=1, group=4),
              dict(threads=64, bulk=1, pdl=1, group=16)]
  for bsuite_id, batch in (('deep_sea/11', 65536), ('deep_sea/20', 32768), ('deep_sea/3', 262144), ('deep_sea/0', 262144)):
    size = bsuite_b200.sweep.SETTINGS[bsuite_id]['size']
    bytes_per = 4 * size * size + 24
    reference = None
    gen = torch.Generator(device='cuda')
    gen.manual_seed(7)
    acts = torch.randint(0, 2, (64, batch), device='cuda', dtype=torch.int32, generator=gen)
    for v in variants:
      os.environ['BSB_BLOCK_THREADS'] = str(v['threads'])
      os.environ['BSB_DEEP_SEA_BULK'] = str(v['bulk'])
      os.environ['BSB_PDL'] = str(v['pdl'])
      os.environ['BSB_DEEP_SEA_GROUP'] = str(v['group'])
      env = bsuite_b200.load_from_id(bsuite_id, batch=batch, device='cuda', seed=0)
      ring_n = max(2, int(400e6 // (batch * size * size * 4)) + 1)
      ring = [env.make_buffers() for _ in range(ring_n)]
      check = env.make_buffers(40)
      ts = env.rollout(40, actions=acts[:40], out=check)
      single = [env.step(acts[40 + i]) for i in range(3)]
      got = [ts.step_type.clone(), ts.reward.clone(), ts.observation.sum(dim=(2, 3)).clone(), ts.observation[-1].clone(),
             single[-1].observation.clone(), single[-1].reward.clone()]
      if reference is None:
        reference = got
      else:
        for a, b in zip(reference, got):
          assert torch.equal(a, b), f'{bsuite_id} {v} differs from the first variant'
      del check, ts, single
      step_s = timeit(lambda i: env.step(acts[i % 64], out=ring[i % ring_n]), args.steps)
      T = 8
      rbuf = env.make_buffers(T)
      roll_s = timeit(lambda i: env.rollout(T, out=rbuf), 8, warm=2) / T
      row = dict(bsuite_id=bsuite_id, size=size, batch=batch, **v,
                 step_us=step_s * 1e6, step_gbs=batch * bytes_per / step_s / 1e9,
                 rollout_us=roll_s * 1e6, rollout_gbs=batch * bytes_per / roll_s / 1e9)
      rows.append(row)
      print(f"{bsuite_id:14s} threads={v['threads']:<4d} bulk={v['bulk']} group={v['group']:<2d} pdl={v['pdl']}  step {row['step_us']:7.1f} us "
            f"{row['step_gbs']:6.0f} GB/s | rollout {row['rollout_us']:7.1f} us/step {row['rollout_gbs']:6.0f} GB/s", flush=True)
      env.close()
      del ring, rbuf
      torch.cuda.empty_cache()
  if args.out:
    with open(args.out, 'w') as fh:
      for r in rows:
        fh.write(json.dumps(r) + '\n')


if __name__ == '__main__':
  main()
