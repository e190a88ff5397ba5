#!/usr/bin/env python
"""Times `bsb_to_image` (the interpolating branch of ImageObservation / to_image) on the GPU.

    python tools/bench_image.py [--batch 4096] [--launches 200] [--out results.jsonl]

Per workload (bsuite_id at B lanes) and target shape it prints one JSON line with
  * us_per_call     -- CUDA-event time of one bsb_to_image launch, averaged over --launches after a warm-up;
  * write_GBps      -- bytes the call must write (B * H * W * C * 4) over that time, and `of_3.35TBps`, its fraction
                       of the H100 SXM data-sheet HBM bandwidth;
  * images_per_s    -- ImageObservation(env).step(actions) over --steps steps: env step + resize, B images per step;
  * interpolate_us  -- for context only, F.interpolate(mode='bilinear') + expand(...).contiguous() on the same shapes.
                       It is NOT output-equal (it clamps at the border where skimage reflects, and has no
                       anti-aliasing filter).
The card's name and power limit are read in the same run.  mnist uses a synthetic dataset in a temporary directory.
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

import bsuite_b200  # noqa: E402
from bsuite_b200 import adapters, datasets, imaging  # noqa: E402

WORKLOADS = ('catch/0', 'deep_sea/11', 'mnist/0', 'cartpole/0', 'umbrella_distract/22')
TARGETS = ((84, 84, 4), (84, 84))
PEAK_BYTES_PER_S = 3.35e12


def card():
  props = torch.cuda.get_device_properties(0)
  info = {'gpu': props.name, 'sms': props.multi_processor_count}
  try:
    bus = '%04x:%02x:%02x.0' % (props.pci_domain_id, props.pci_bus_id, props.pci_device_id)
    out = subprocess.run(['nvidia-smi', '-i', bus, '--query-gpu=name,power.limit', '--format=csv,noheader'],
                         capture_output=True, text=True, timeout=30).stdout.strip()
    info['nvidia_smi'] = out
  except Exception as error:  # pylint: disable=broad-except
    info['nvidia_smi'] = f'unavailable: {error}'
  return info


def time_ms(fn, repeats):
  start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  start.record()
  for _ in range(repeats):
    fn()
  end.record()
  end.synchronize()
  return start.elapsed_time(end) / repeats


def main():
  parser = argparse.ArgumentParser()
  parser.add_argument('--batch', type=int, default=4096)
  parser.add_argument('--launches', type=int, default=200)
  parser.add_argument('--steps', type=int, default=100)
  parser.add_argument('--out', default=None)
  args = parser.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit('bench_image.py measures the CUDA kernel: no GPU found')
  os.environ[datasets.ENV_VAR] = datasets.write_synthetic_mnist(tempfile.mkdtemp(prefix='bsb_bench_mnist_'), 256, 16, 0)
  conditions = card()
  print(json.dumps(conditions), flush=True)
  lines = [conditions]
  B = args.batch
  for bsuite_id in WORKLOADS:
    raw = bsuite_b200.load_from_id(bsuite_id, batch=B, device='cuda', seed=1)
    actions = torch.as_tensor(raw.random_actions(args.steps, action_seed=1, first_step=0)).cuda()
    raw.reset()
    obs = raw.step(actions[0]).observation.clone()
    plane = tuple(obs.shape[1:])
    plane = (1,) + plane if len(plane) == 1 else plane
    planes = obs.reshape((B,) + plane).contiguous()
    for target in TARGETS:
      channels = 1 if len(target) == 2 else target[2]
      plan = imaging.plan_for(plane, target[:2], channels, planes.device)
      out = torch.empty((B,) + target, device='cuda')
      stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
      call = lambda: plan(planes, out, stream)  # noqa: E731
      for _ in range(20):
        call()
      ms = time_ms(call, args.launches)
      written = B * target[0] * target[1] * channels * 4
      env = adapters.ImageObservation(bsuite_b200.load_from_id(bsuite_id, batch=B, device='cuda', seed=1), target)
      env.reset()
      for t in range(5):
        env.step(actions[t])
      step_ms = time_ms(lambda: env.step(actions[7]), args.steps)
      env.close()
      src = planes.unsqueeze(1)
      ref = lambda: F.interpolate(src, size=target[:2], mode='bilinear', align_corners=False).reshape(  # noqa: E731
          (B,) + target[:2] + (1,)).expand((B,) + target[:2] + (channels,)).contiguous()
      for _ in range(5):
        ref()
      ref_ms = time_ms(ref, args.launches)
      line = {'workload': bsuite_id, 'batch': B, 'plane': list(plane), 'target': list(target),
              'launches': args.launches, 'us_per_call': round(ms * 1e3, 2), 'bytes_written': written,
              'write_GBps': round(written / (ms * 1e-3) / 1e9, 1),
              'of_3.35TBps': round(written / (ms * 1e-3) / PEAK_BYTES_PER_S, 3),
              'step_plus_resize_us': round(step_ms * 1e3, 2), 'images_per_s': round(B / (step_ms * 1e-3)),
              'interpolate_us_not_output_equal': round(ref_ms * 1e3, 2)}
      print(json.dumps(line), flush=True)
      lines.append(line)
    raw.close()
  if args.out:
    with open(args.out, 'w') as f:
      for line in lines:
        f.write(json.dumps(line) + '\n')


if __name__ == '__main__':
  main()
