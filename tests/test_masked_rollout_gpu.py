"""Masked rollouts on the device (masked_kernel, T steps per launch) against the host path."""
import numpy as np
import pytest
import torch

import bsuite_b200
from bsuite_b200 import analysis
from bsuite_b200 import rollouts
from tests import conftest as cf
from tests import test_masked as tm
from tests import test_masked_gpu as tmg
from tests import test_masked_rollout as tr

pytestmark = pytest.mark.gpu


def compare_out(case, out_d, out_h, where=''):
  """Every field of two [T, ...] buffers: step types, discounts and actions bit for bit, as are observations of the
  integer-dynamics families; rewards of those within 1e-12 relative (RewardNoise draws through log()); float-dynamics
  families within FLOAT_TOL.  Unwritten entries hold the sentinel on both sides."""
  exact = case[0] not in ('Cartpole', 'CartpoleSwingup', 'MountainCar')
  for name in tr.FIELDS:
    a, b = getattr(out_d, name), getattr(out_h, name)
    if a is None:
      assert b is None
      continue
    a = a.cpu()
    if name in ('step_type', 'discount', 'actions') or (exact and name != 'reward'):
      assert torch.equal(a, b), f'{name} {where}'
    else:
      tol = 1e-12 if exact else cf.FLOAT_TOL
      torch.testing.assert_close(a.double(), b.double(), rtol=tol, atol=tol, msg=f'{name} {where}')


def compare_acc(case, dev, host):
  exact = case[0] not in ('Cartpole', 'CartpoleSwingup', 'MountainCar')
  acc_d, acc_h = tm.accumulators(dev), tm.accumulators(host)
  for key in acc_h:
    tol = 1e-12 if exact else cf.FLOAT_TOL
    torch.testing.assert_close(acc_d[key], acc_h[key], rtol=tol, atol=tol, msg=key)


def run_launches(case, dev, host, launches, action_seed=5):
  same_step = case[2] == 'SAME_STEP'
  for k, launch in enumerate(launches):
    T = launch[0]
    out_d = dev.make_buffers(T, with_actions=True, final_observation=same_step)
    out_h = host.make_buffers(T, with_actions=True, final_observation=same_step)
    left_d = tr.rollout_launch(dev, launch, out_d, action_seed)
    left_h = tr.rollout_launch(host, launch, out_h, action_seed)
    compare_out(case, out_d, out_h, f'in launch {k}')
    if left_h is not None:
      assert np.array_equal(left_d, left_h), f'budgets after launch {k}'
  assert dev.steps_done == host.steps_done
  compare_acc(case, dev, host)


@pytest.mark.parametrize('case', tmg.masked_kernel_cases(), ids=lambda c: '-'.join(c))
def test_every_masked_rollout_kernel_matches_the_host_path(case, mnist_dir):
  """97 lanes: three full warps and a partial one; budgets of 0-3 episodes end at different steps of one warp."""
  del mnist_dir
  dev, host = tmg.make_env(case, 'cuda', 97), tmg.make_env(case, 'cpu', 97)
  run_launches(case, dev, host, tr.make_launches(dev.batch, dev.num_actions, seed=dev.batch + len(case[0])))


@pytest.mark.parametrize('bsuite_id,case', [('deep_sea/11', ('DeepSea', 'float', 'NEXT_STEP', 'philox')),
                                            ('catch/0', ('Catch', 'float', 'NEXT_STEP', 'philox')),
                                            ('cartpole/0', ('Cartpole', 'float', 'NEXT_STEP', 'philox'))])
def test_large_batch_matches_the_host_path(bsuite_id, case):
  """B = 4 099; deep_sea's observations in compressible memory where the device offers it (obs_memory)."""
  kw = dict(batch=4099, seed=5, track_episodes=True, record_rows=True)
  dev = bsuite_b200.load_from_id(bsuite_id, device='cuda', **kw)
  host = bsuite_b200.load_from_id(bsuite_id, device='cpu', **kw)
  launches = tr.make_launches(4099, dev.num_actions, seed=2, densities=(1.0, 0.5, 0.01, 0.5), steps=(9, 16, 4, 12))
  run_launches(case, dev, host, launches)


def test_captured_masked_rollout_counts_budgets_down_across_replays():
  B, T, seed = 97, 6, 6
  kw = dict(batch=B, seed=seed, track_episodes=True, record_rows=True, autoreset='same_step')
  dev = bsuite_b200.load_from_id('bandit/0', device='cuda', **kw)
  host = bsuite_b200.load_from_id('bandit/0', device='cpu', **kw)
  out_d, out_h = dev.make_buffers(T, with_actions=True), host.make_buffers(T, with_actions=True)
  mask = torch.ones(B, dtype=torch.bool, device='cuda')
  left = torch.full((B,), 40, dtype=torch.int64, device='cuda')
  left_h = left.cpu()
  dev.rollout(T, out=out_d, mask=mask, episodes_left=left)        # module loading happens outside the capture
  host.rollout(T, out=out_h, mask=mask.cpu(), episodes_left=left_h)
  torch.cuda.synchronize()
  graph = torch.cuda.CUDAGraph()
  with torch.cuda.graph(graph, capture_error_mode='thread_local'):
    dev.rollout(T, action_seed=2, out=out_d, mask=mask, episodes_left=left)
  torch.cuda.synchronize()
  rng = np.random.default_rng(0)
  for r in range(10):
    m = torch.as_tensor(rng.random(B) < (0.5, 0.03, 1.0, 0.0, 0.9)[r % 5])
    mask.copy_(m)
    if r == 4:                               # new budgets between replays, some of them zero
      budgets = torch.as_tensor(rng.integers(0, 8, B).astype(np.int64))
      left.copy_(budgets)
      left_h.copy_(budgets)
    tr.fill(out_d)
    tr.fill(out_h)
    graph.replay()
    host.rollout(T, action_seed=2, out=out_h, mask=m, episodes_left=left_h)
    torch.cuda.synchronize()
    assert torch.equal(left.cpu(), left_h), f'budgets after replay {r}'
    for name in ('observation', 'reward', 'discount', 'step_type', 'actions'):
      assert torch.equal(getattr(out_d, name).cpu(), getattr(out_h, name)), f'{name} after replay {r}'
    if r % 3 == 2:                           # eager masked rollouts between replays
      dev.rollout(T, action_seed=9, out=out_d, mask=mask, episodes_left=left)
      host.rollout(T, action_seed=9, out=out_h, mask=m, episodes_left=left_h)
  torch.cuda.synchronize()
  assert torch.equal(left.cpu(), left_h)
  assert dev.steps_done == host.steps_done
  for key, value in tm.accumulators(host).items():
    assert torch.equal(tm.accumulators(dev)[key], value), key


def test_invalid_action_flag_only_for_active_lanes():
  env = bsuite_b200.load_from_id('catch/0', batch=64, device='cuda', seed=0)
  out = env.make_buffers(4)
  mask = torch.zeros(64, dtype=torch.bool, device='cuda')
  mask[:40] = True
  left = torch.ones(64, dtype=torch.int64, device='cuda')
  left[30:40] = 0                            # masked in, but no budget: never active
  env.reset(out=env.make_buffers())
  env.invalid_actions_seen()
  actions = torch.ones((4, 64), dtype=torch.int32, device='cuda')
  actions[:, 30:] = 99                       # inactive lanes: never read
  env.rollout(4, actions=actions, out=out, mask=mask, episodes_left=left)
  assert not env.invalid_actions_seen()
  actions[2, 3] = -4
  env.rollout(4, actions=actions, out=out, mask=mask, episodes_left=left)
  assert env.invalid_actions_seen()


def test_run_random_episodes_on_a_cuda_pack_matches_the_host_path():
  kw = dict(seed=1, track_episodes=True, record_rows=True)
  dev = bsuite_b200.load_experiment('catch', 40, device='cuda', **kw)
  host = bsuite_b200.load_experiment('catch', 40, device='cpu', **kw)
  specs = list(dev._pack[1]) + [spec for spec in host._pack[1] if all(spec is not s for s in dev._pack[1])]
  budgets = [spec.bsuite_num_episodes for spec in specs]
  small = [2 + k % 5 for k in range(len(dev._pack[1]))]
  for k, spec in enumerate(specs):             # a short run: each setting's budget lowered in place
    spec.bsuite_num_episodes = small[k % len(small)]
  try:
    calls_d = rollouts.run_random_episodes(dev, action_seed=4, steps_per_launch=16)
    calls_h = rollouts.run_random_episodes(host, action_seed=4, steps_per_launch=16)
  finally:
    for spec, n in zip(specs, budgets):
      spec.bsuite_num_episodes = n
  assert calls_d == calls_h
  acc_d, acc_h = tm.accumulators(dev), tm.accumulators(host)
  for key in acc_h:
    assert torch.equal(acc_d[key], acc_h[key]), key
  a, b = analysis.bsuite_score(dev), analysis.bsuite_score(host)
  assert torch.equal(a.score.cpu().view(torch.int64), b.score.view(torch.int64))
  assert torch.equal(a.finished.cpu(), b.finished)
