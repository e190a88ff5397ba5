#!/usr/bin/env python
"""A workload for compute-sanitizer that exercises the PERSISTENT deep_sea path (dynamic chunk counter, grouped
TMA bulk stores with L2 hints, PDL) plus the catch / row bulk emitters and the to_image kernel at a size the
sanitizer finishes quickly.

    compute-sanitizer --tool memcheck  python tools/sanitize_check.py
    compute-sanitizer --tool racecheck python tools/sanitize_check.py
"""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
import bsuite_b200


def split_steps():
  """Host steps left in flight (BSB_HOST_NO_WAIT) on 2 / 3 handles driven round-robin, against one ordinary
  environment."""
  from bsuite_b200 import rollouts
  for bsuite_id, batch, parts in (('deep_sea/11', 12000 + 5, 3), ('deep_sea_stochastic/3', 9000, 2)):
    group = rollouts.HostParts(bsuite_id, batch, device='cuda', seed=3, track_episodes=True, parts=parts)
    twin = bsuite_b200.load_from_id(bsuite_id, batch=batch, device='cuda', seed=3, track_episodes=True)
    bounds = [0]
    for size in group.sizes:
      bounds.append(bounds[-1] + size)
    T = 5
    acts = torch.as_tensor(twin.random_actions(T, action_seed=1, first_step=0))
    rows = [acts[:, bounds[p]:bounds[p + 1]].contiguous().pin_memory() for p in range(parts)]
    group.reset(); twin.reset()
    want = [twin.step(acts[t].cuda(), out=twin.make_buffers()) for t in range(T)]
    torch.cuda.synchronize()

    def check(p, t, ts, obs):
      lanes = slice(bounds[p], bounds[p + 1])
      torch.cuda.synchronize()
      assert torch.equal(obs, want[t].observation[lanes]) and torch.equal(ts.reward, want[t].reward.cpu()[lanes]) \
          and torch.equal(ts.step_type, want[t].step_type.cpu()[lanes]), (p, t)

    for p in range(parts):
      group.submit(p, rows[p][0])
    for t in range(1, T):
      for p in range(parts):
        check(p, t - 1, *group.collect(p)); group.submit(p, rows[p][t])
    for p in range(parts):
      check(p, T - 1, *group.collect(p))
    print(bsuite_id, batch, f'{parts} parts, round-robin host steps == ordinary steps: True', flush=True)
    group.close(); twin.close()


if '--only-split' in sys.argv:
  split_steps()
  print('sanitize workload (split steps) finished')
  sys.exit(0)

def buffers(env, bsuite_id, plain, num_steps=None):
  """Bulk stores land in `plain` torch.empty memory; the other leg writes where the store path changes: the
  compressible pool (make_buffers) for deep_sea, whose large batches then compare each tile with the destination
  (single steps) or take 16-byte streaming stores (rollouts), and an
  observation one float past a 16-byte boundary (vector / scalar stores) for every other family."""
  out = env.make_buffers(num_steps)
  n = out.observation.numel()
  if plain:
    out.observation = torch.empty(out.observation.shape, device='cuda')
  elif not bsuite_id.startswith('deep_sea'):
    out.observation = torch.empty(n + 4, device='cuda')[1:n + 1].view(out.observation.shape)
  return out


for bsuite_id, batch in (('deep_sea/11', 20000), ('deep_sea_stochastic/3', 40001), ('catch_noise/0', 5000), ('cartpole/0', 3000),
                         ('umbrella_length/3', 2000), ('umbrella_distract/22', 1500), ('mnist/0', 1500), ('mnist/0', 30000)):
  if bsuite_id.startswith('mnist'):
    from bsuite_b200 import datasets
    os.environ[datasets.ENV_VAR] = datasets.write_synthetic_mnist('/tmp/bsb_sanitize_mnist', 256, 16, 0)
  results = []
  for plain in (True, False):
    env = bsuite_b200.load_from_id(bsuite_id, batch=batch, device='cuda', seed=3, track_episodes=True)
    acts = torch.as_tensor(env.random_actions(4, action_seed=1, first_step=0)).cuda()
    outs = [env.step(acts[i], out=buffers(env, bsuite_id, plain)).observation.clone() for i in range(4)]
    ts = env.rollout(3, action_seed=2, out=buffers(env, bsuite_id, plain, 3))
    results.append(outs + [ts.observation.clone(), ts.reward.clone(), ts.step_type.clone()])
    torch.cuda.synchronize()
    env.close()
  same = all(torch.equal(a, b) for a, b in zip(*results))
  print(bsuite_id, batch, 'bulk == vector:', same, flush=True)
  assert same
# Reduced observation dtypes: uint8 deep_sea tiles (16-lane groups) and bfloat16 catch boards, against float32 twins.
for bsuite_id, batch, dtype in (('deep_sea/11', 20000, torch.uint8), ('catch/0', 5001, torch.bfloat16)):
  env = bsuite_b200.load_from_id(bsuite_id, batch=batch, device='cuda', seed=3, obs_dtype=dtype)
  twin = bsuite_b200.load_from_id(bsuite_id, batch=batch, device='cuda', seed=3)
  acts = torch.as_tensor(env.random_actions(4, action_seed=1, first_step=0)).cuda()
  for i in range(4):
    assert torch.equal(env.step(acts[i]).observation, twin.step(acts[i]).observation.to(dtype))
  assert torch.equal(env.rollout(3, action_seed=2).observation, twin.rollout(3, action_seed=2).observation.to(dtype))
  print(bsuite_id, batch, dtype, '== float32 twin converted: True', flush=True)
  env.close(); twin.close()
# Graph-safe mode: device clock, chunk counter re-armed by the last CTA, the deterministic two-stage reduction.
for bsuite_id, batch in (('deep_sea/11', 20000), ('catch/0', 5000)):
  env = bsuite_b200.load_from_id(bsuite_id, batch=batch, device='cuda', seed=3, track_episodes=True)
  twin = bsuite_b200.load_from_id(bsuite_id, batch=batch, device='cuda', seed=3, track_episodes=True)
  graphed = env.capture(2, sample_actions=True, action_seed=5)
  for _ in range(3):
    got = graphed.replay()
    want = twin.rollout(2, action_seed=5)
    assert torch.equal(got.observation, want.observation) and torch.equal(got.reward, want.reward)
  env.step(torch.zeros(batch, dtype=torch.int32, device='cuda'))
  twin.step(torch.zeros(batch, dtype=torch.int32, device='cuda'))
  assert torch.equal(env.episode_stat_sums(), twin.episode_stat_sums()) and env.steps_done == twin.steps_done == 7
  print(bsuite_id, batch, 'graph replay == eager: True', flush=True)
  env.close(); twin.close()
# Host-driven steps: completion through the pinned mailbox, out-of-range actions.
for bsuite_id, batch in (('deep_sea/11', 20000), ('catch/0', 3000), ('mnist/0', 1500)):
  env = bsuite_b200.load_from_id(bsuite_id, batch=batch, device='cuda', seed=3, track_episodes=True)
  twin = bsuite_b200.load_from_id(bsuite_id, batch=batch, device='cuda', seed=3, track_episodes=True)
  host = env.make_host_buffers()
  acts = torch.as_tensor(env.random_actions(6, action_seed=1, first_step=0)).pin_memory()
  env.reset(); twin.reset()
  for t in range(6):
    got, obs = env.step_host(acts[t], host)
    want = twin.step(acts[t].cuda())
    torch.cuda.synchronize()
    assert torch.equal(obs, want.observation) and torch.equal(got.reward, want.reward.cpu()) and torch.equal(got.step_type, want.step_type.cpu())
  bad = acts[0].cuda().clone(); bad[5] = 99
  env.step(bad); twin.step(bad.clamp(max=env.num_actions - 1))
  assert env.invalid_actions_seen() and torch.equal(env.episode_stat_sums(), twin.episode_stat_sums())
  print(bsuite_id, batch, 'host-driven steps == ordinary steps: True', flush=True)
  env.close(); twin.close()
split_steps()
# Masked calls (masked_kernel): warp-written tiles / boards / rows of a lane subset, partial warps, same-step final
# observations and a ragged pack, against the host path.
for bsuite_id, batch, kw in (('deep_sea/11', 1001, {}), ('catch/0', 997, dict(autoreset='same_step')),
                             ('umbrella_distract/3', 501, {}), ('mnist/0', 333, dict(obs_dtype='bfloat16'))):
  plan = [(kind, torch.rand(batch, generator=torch.Generator().manual_seed(c)) < (0.5, 0.03, 1.0)[c % 3])
          for c, kind in enumerate(('reset', 'step', 'step', 'step', 'reset', 'step'))]
  got = []
  for device in ('cuda', 'cpu'):
    env = bsuite_b200.load_from_id(bsuite_id, batch=batch, device=device, seed=3, track_episodes=True, **kw)
    out = env.make_buffers(final_observation='autoreset' in kw)
    out.observation.fill_(5)
    for kind, mask in plan:
      if kind == 'reset':
        env.reset(out=out, mask=mask.to(device))
      else:
        env.step(torch.ones(batch, dtype=torch.int32, device=device), out=out, mask=mask.to(device))
    got.append([out.observation.cpu(), out.reward.cpu(), env.episode_stat_sums().cpu()])
    env.close()
  assert all(torch.equal(a, b) for a, b in zip(*got))
  print(bsuite_id, batch, 'masked calls == host path: True', flush=True)
# Masked rollouts (masked_kernel again): the same workloads as T steps per launch, lanes stopping at their own
# budgets mid-launch, sampled actions written to actions_out, against the host path.
for bsuite_id, batch, kw in (('deep_sea/11', 1001, {}), ('catch/0', 997, dict(autoreset='same_step')),
                             ('umbrella_distract/3', 501, {}), ('mnist/0', 333, dict(obs_dtype='bfloat16'))):
  gen = torch.Generator().manual_seed(4)
  mask = torch.rand(batch, generator=gen) < 0.7
  budgets = torch.randint(0, 3, (batch,), generator=gen, dtype=torch.int64)
  got = []
  for device in ('cuda', 'cpu'):
    env = bsuite_b200.load_from_id(bsuite_id, batch=batch, device=device, seed=3, track_episodes=True, **kw)
    out = env.make_buffers(12, with_actions=True, final_observation='autoreset' in kw)
    for buf in (out.observation, out.reward, out.discount, out.step_type, out.actions):
      buf.fill_(5)                           # entries of steps a lane sits out are never written
    left = budgets.clone().to(device)
    for _ in range(3):
      env.rollout(12, action_seed=1, out=out, mask=mask.to(device), episodes_left=left)
    got.append([out.observation.cpu(), out.reward.cpu(), out.actions.cpu(), left.cpu()] +
               [v.cpu() for v in env.episode_stats().values()])      # per lane: sums over lanes may round differently
    env.close()
  assert all(torch.equal(a, b) for a, b in zip(*got))
  print(bsuite_id, batch, 'masked rollouts == host path: True', flush=True)
# One-launch reduction over several environments and a whole lock-step in one graph.
from bsuite_b200 import suite
ids = ['catch/0', 'deep_sea/0', 'bandit_noise/0', 'cartpole/0', 'mnist/0', 'umbrella_length/0']
a, b = suite.SweepBatch(ids, lanes=300, device='cuda', seed=1), suite.SweepBatch(ids, lanes=300, device='cuda', seed=1, ring=2)
graphed = a.capture(1, lock_steps=2)
for _ in range(3):
  got, want = graphed.replay(), [b.rollout(1), b.rollout(1)]
  torch.cuda.synchronize()
  assert all(torch.equal(got[i][k].observation, want[i][k].observation) for i in range(2) for k in ids)
assert torch.equal(a.gather_returns(), b.local_returns().unsqueeze(0))
print('sweep graph == eager, one-launch reduction == per-id reductions: True', flush=True)
a.close(); b.close()
# bsb_to_image: staged and unstaged planes, bulk stores and the unaligned streaming-store fallback.
from bsuite_b200 import adapters
for plane, target, offset in (((10, 5), (84, 84, 4), 0), ((28, 28), (16, 16), 1), ((130, 100), (90, 70, 3), 1)):
  planes = torch.randn((300,) + plane, device='cuda')
  want = adapters.to_image(target, planes.cpu(), batch_dims=1)
  got = adapters.to_image(target, planes, batch_dims=1)
  buf = torch.empty(want.numel() + offset, device='cuda')
  import ctypes
  from bsuite_b200 import imaging
  imaging.plan_for(plane, target[:2], (target[2] if len(target) > 2 else 1), planes.device)(
      planes, buf[offset:], ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
  torch.cuda.synchronize()
  assert torch.equal(got.cpu(), want) and torch.equal(buf[offset:].cpu().view(want.shape), want)
  print(plane, '->', target, 'offset', offset, 'CUDA to_image == host path: True', flush=True)
print('sanitize workload finished')
