#!/usr/bin/env python
"""Where the time of one host-driven step goes (deep_sea N=32, B=65536, one GPU).

    python tools/e2e_breakdown.py [bsuite_id] [batch]

Rows: the kernel rate (launches queued), a device-resident loop that synchronises after every step, then the
host-buffer call `BatchedEnvironment.step_host` (pinned actions in, pinned scalars out; two-phase, scalars first,
for deep_sea) through the Python face and through bare ctypes calls with prebuilt arguments (what a C caller of the
ABI pays), and its staged copies from pageable buffers.
"""
import ctypes
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
import bsuite_b200
from bsuite_b200 import _lib

BSUITE_ID = sys.argv[1] if len(sys.argv) > 1 else 'deep_sea/11'
B = int(sys.argv[2]) if len(sys.argv) > 2 else 65536


def timed(fn, n=300):
  for i in range(20):
    fn(i)
  torch.cuda.synchronize()
  t0 = time.perf_counter()
  for i in range(n):
    fn(i)
  torch.cuda.synchronize()
  return (time.perf_counter() - t0) / n * 1e6


env = bsuite_b200.load_from_id(BSUITE_ID, batch=B, device='cuda', seed=0, track_episodes=True)
ring = [env.make_buffers() for _ in range(4)]
n_act = env.num_actions
dev_acts = torch.randint(0, n_act, (64, B), device='cuda', dtype=torch.int32)
rows = [dev_acts[i] for i in range(64)]
pin = torch.randint(0, n_act, (64, B), dtype=torch.int32).pin_memory()
prow = [pin[i] for i in range(64)]
host = env.make_host_buffers()

print(f'{BSUITE_ID} B={B}')
print(f'device actions, launches queued (kernel rate)            {timed(lambda i: env.step(rows[i % 64], out=ring[i % 4])):7.1f} us/step')


def dev_sync(i):
  env.step(rows[i % 64], out=ring[i % 4])
  torch.cuda.synchronize()


print(f'device actions, synchronise after every step             {timed(dev_sync):7.1f} us/step')


def variants(e, label):
  lib, handle = e._lib, e._handle.ptr          # pylint: disable=protected-access
  houts = host.as_outputs()
  acts = [ctypes.c_void_p(p.data_ptr()) for p in prow]
  obs = [ctypes.c_void_p(r.observation.data_ptr()) for r in ring]
  ref = ctypes.byref(houts)
  py = timed(lambda i: e.step_host(prow[i % 64], host, out=ring[i % 4]))
  raw = timed(lambda i: lib.bsb_step_host(handle, acts[i % 64], ref, obs[i % 4], None, 0))
  print(f'step_host {label:34s}  python {py:6.1f}  ctypes {raw:6.1f} us/step')


variants(env, 'mailbox + two-phase')
page = [torch.empty(B, dtype=torch.int32).copy_(row) for row in prow[:4]]      # pageable host memory
page_host = type(host)(observation=None, **{f: torch.empty(getattr(host, f).shape, dtype=getattr(host, f).dtype)
                                              for f in ('reward', 'discount', 'step_type')})
print(f'step_host staged copies (pageable buffers)               {timed(lambda i: env.step_host(page[i % 4], page_host, out=ring[i % 4])):7.1f} us/step')
