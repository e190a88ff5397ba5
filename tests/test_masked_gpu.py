"""Masked resets and steps on the device (masked_kernel): against the host path and against separate device
handles."""
import numpy as np
import pytest
import torch

import bsuite_b200
from bsuite_b200 import build as bsb_build
from bsuite_b200 import sweep
from tests import conftest as cf
from tests import test_masked as tm

pytestmark = pytest.mark.gpu

FAMILY_IDS = {'DeepSea': 'deep_sea/1', 'Catch': 'catch/0', 'Cartpole': 'cartpole/0',
              'CartpoleSwingup': 'cartpole_swingup/2', 'MountainCar': 'mountain_car_noise/1', 'MemoryChain': 'memory_len/3',
              'Bandit': 'bandit_noise/2', 'UmbrellaChain': 'umbrella_distract/4', 'DiscountingChain': 'discounting_chain/0',
              'Mnist': 'mnist/0'}
PACKED_EXPERIMENTS = {'Catch': 'catch_scale', 'Cartpole': 'cartpole_noise', 'CartpoleSwingup': 'cartpole_swingup',
                      'MountainCar': 'mountain_car_scale', 'MemoryChain': 'memory_len', 'Bandit': 'bandit_noise',
                      'UmbrellaChain': 'umbrella_length', 'DiscountingChain': 'discounting_chain', 'Mnist': 'mnist_noise'}
RAGGED_EXPERIMENTS = {'DeepSea': 'deep_sea', 'MemoryChain': 'memory_size', 'UmbrellaChain': 'umbrella_distract'}
OBS = {'float': 'float32', 'Bf16': 'bfloat16', 'uint8_t': 'uint8'}


def masked_kernel_cases():
  """One case per variant of the list and bit source, (family, O, mode, bit source): its masked_kernel instantiations
  (masked resets and steps here, masked rollouts in test_masked_rollout_gpu)."""
  cases = []
  for variants in bsb_build.variant_list().values():
    for family, obs, mode, mt, _ in variants:
      cases.append((family, obs, mode, 'philox'))
      if mt:
        cases.append((family, obs, mode, 'mt19937'))
  return cases


def make_env(case, device, batch):
  family, obs, mode, rng = case
  kw = dict(track_episodes=True, record_rows=rng == 'philox', seed=3)
  if mode in ('PACKED', 'RAGGED'):
    name = (PACKED_EXPERIMENTS if mode == 'PACKED' else RAGGED_EXPERIMENTS)[family]
    lanes = max(1, batch // len(sweep.BY_EXPERIMENT[name]))
    return bsuite_b200.load_experiment(name, lanes, device=device, ragged=mode == 'RAGGED', **kw)
  return bsuite_b200.load_from_id(FAMILY_IDS[family], batch=batch, device=device, rng=rng, obs_dtype=OBS[obs],
                                  autoreset='same_step' if mode == 'SAME_STEP' else 'next_step', **kw)


def compare(case, got_dev, got_host, acc_dev, acc_host):
  """Observations, step types and discounts bit for bit (float-dynamics families: within FLOAT_TOL); rewards and the
  accumulators that sum them within 1e-12 relative (RewardNoise draws through log(): CUDA's and glibc's may differ in
  the last ulp), float-dynamics families within FLOAT_TOL."""
  exact = case[0] not in ('Cartpole', 'CartpoleSwingup', 'MountainCar')
  for name in tm.FIELDS:
    for c, (row_d, row_h) in enumerate(zip(got_dev[name], got_host[name])):
      for i, (a, b) in enumerate(zip(row_d, row_h)):
        if a is None or b is None:
          assert a is None and b is None
          continue
        if name in ('step_type', 'discount') or (exact and name != 'reward'):
          assert torch.equal(a, b), f'{name} of lane {i} at call {c}'
        elif exact:
          torch.testing.assert_close(a.double(), b.double(), rtol=1e-12, atol=1e-12, msg=f'{name} of lane {i} at call {c}')
        else:
          torch.testing.assert_close(a.double(), b.double(), rtol=0, atol=cf.FLOAT_TOL, msg=f'{name} of lane {i} at call {c}')
  for key in acc_host:
    tol = 1e-12 if exact else cf.FLOAT_TOL
    torch.testing.assert_close(acc_dev[key], acc_host[key], rtol=tol, atol=tol, msg=key)


def run_both(case, batch, calls=24):
  dev = make_env(case, 'cuda', batch)
  host = make_env(case, 'cpu', batch)
  plan = tm.make_plan(dev.batch, calls, dev.num_actions, seed=dev.batch + len(case[0]), densities=(0.5, 1.0, 0.03, 0.0, 0.7))
  same_step = case[2] == 'SAME_STEP'
  got_dev = tm.drive(dev, plan, final_observation=same_step)
  got_host = tm.drive(host, plan, final_observation=same_step)
  compare(case, got_dev, got_host, tm.accumulators(dev), tm.accumulators(host))
  assert dev.steps_done == host.steps_done == calls
  return dev, plan, got_dev


@pytest.mark.parametrize('case', masked_kernel_cases(), ids=lambda c: '-'.join(c))
def test_every_masked_kernel_matches_the_host_path(case, mnist_dir):
  del mnist_dir
  run_both(case, 97)


def test_gpu_cases_cover_every_masked_kernel_of_the_list():
  """Each variant of the list, times its bit sources, has a case above, and with it both masked_kernel instantiations."""
  cases = masked_kernel_cases()
  want = sum(1 + int(mt) for variants in bsb_build.variant_list().values() for _, _, _, mt, _ in variants)
  assert len(set(cases)) == len(cases) == want
  for family, obs, mode, _ in cases:
    if mode == 'PACKED':
      assert family in PACKED_EXPERIMENTS
    elif mode == 'RAGGED':
      assert family in RAGGED_EXPERIMENTS
    else:
      assert family in FAMILY_IDS and obs in OBS


@pytest.mark.parametrize('bsuite_id', ['deep_sea/11', 'catch/0', 'cartpole/0'])
def test_large_batch_matches_separate_device_handles(bsuite_id):
  """B = 4096 on the device: lanes against one-lane device handles (a sample of lanes), bit for bit."""
  B, seed = 4096, 5
  env = bsuite_b200.load_from_id(bsuite_id, batch=B, device='cuda', seed=seed, track_episodes=True, record_rows=True)
  plan = tm.make_plan(B, 12, env.num_actions, seed=1, densities=(1.0, 0.5, 0.01, 0.5))
  got = tm.drive(env, plan)
  lanes = [0, 31, 32, 1000, 2047, 4095]
  tm.check_against_one_lane(env, plan, got, lambda i: bsuite_b200.load_from_id(
      bsuite_id, batch=1, device='cuda', seed=seed, lane_offset=i, track_episodes=True, record_rows=True), lanes=lanes)


def test_partial_warps_match_separate_device_handles():
  B, seed = 97, 2
  env = bsuite_b200.load_from_id('umbrella_distract/3', batch=B, device='cuda', seed=seed, track_episodes=True,
                                 record_rows=True)
  plan = tm.make_plan(B, 30, env.num_actions, seed=4)
  got = tm.drive(env, plan)
  tm.check_against_one_lane(env, plan, got, lambda i: bsuite_b200.load_from_id(
      'umbrella_distract/3', batch=1, device='cuda', seed=seed, lane_offset=i, track_episodes=True,
      record_rows=True), lanes=[0, 5, 31, 32, 64, 96])


def test_deep_sea_in_compressible_memory():
  """deep_sea observation buffers come from compressible memory where the device offers it (obs_memory)."""
  case = ('DeepSea', 'float', 'NEXT_STEP', 'philox')
  dev = bsuite_b200.load_from_id('deep_sea/11', batch=1024, device='cuda', seed=1, track_episodes=True)
  host = bsuite_b200.load_from_id('deep_sea/11', batch=1024, device='cpu', seed=1, track_episodes=True)
  plan = tm.make_plan(1024, 6, 2, seed=3, densities=(1.0, 0.5, 0.01))
  compare(case, tm.drive(dev, plan), tm.drive(host, plan), tm.accumulators(dev), tm.accumulators(host))


def test_captured_graph_of_masked_calls_with_changing_masks():
  B = 97
  dev = bsuite_b200.load_from_id('catch/0', batch=B, device='cuda', seed=6, track_episodes=True, record_rows=True)
  host = bsuite_b200.load_from_id('catch/0', batch=B, device='cpu', seed=6, track_episodes=True, record_rows=True)
  out_d, out_h = dev.make_buffers(), host.make_buffers()
  mask = torch.ones(B, dtype=torch.bool, device='cuda')
  actions = torch.zeros(B, dtype=torch.int32, device='cuda')
  dev.reset(out=out_d, mask=mask)          # module loading happens outside the capture
  dev.step(actions, out=out_d, mask=mask)
  host.reset(out=out_h, mask=mask.cpu())
  host.step(actions.cpu(), out=out_h, mask=mask.cpu())
  torch.cuda.synchronize()
  graph = torch.cuda.CUDAGraph()
  with torch.cuda.graph(graph, capture_error_mode='thread_local'):
    dev.reset(out=out_d, mask=mask)
    dev.step(actions, out=out_d, mask=mask)
  torch.cuda.synchronize()
  # the capture recorded the launches without running them: the host handle saw nothing either
  rng = np.random.default_rng(0)
  for r in range(12):
    m = torch.as_tensor(rng.random(B) < (0.5, 0.03, 1.0, 0.0)[r % 4])
    a = torch.as_tensor(rng.integers(0, 3, B).astype(np.int32))
    mask.copy_(m)
    actions.copy_(a)
    graph.replay()
    host.reset(out=out_h, mask=m)
    host.step(a, out=out_h, mask=m)
    if r % 3 == 2:                          # eager masked calls between replays
      dev.step(actions, out=out_d, mask=mask)
      host.step(a, out=out_h, mask=m)
    torch.cuda.synchronize()
    for name in ('observation', 'reward', 'discount', 'step_type'):
      assert torch.equal(getattr(out_d, name).cpu(), getattr(out_h, name)), f'{name} after replay {r}'
  assert dev.steps_done == host.steps_done
  for key, value in tm.accumulators(host).items():
    assert torch.equal(tm.accumulators(dev)[key], value), key


def test_invalid_action_flag_only_for_active_lanes():
  env = bsuite_b200.load_from_id('catch/0', batch=40, device='cuda', seed=0)
  out = env.make_buffers()
  mask = torch.zeros(40, dtype=torch.bool, device='cuda')
  mask[:20] = True
  env.reset(out=out)
  env.invalid_actions_seen()
  actions = torch.ones(40, dtype=torch.int32, device='cuda')
  actions[20:] = 99                          # inactive lanes: never read
  env.step(actions, out=out, mask=mask)
  assert not env.invalid_actions_seen()
  actions[3] = -4
  env.step(actions, out=out, mask=mask)
  assert env.invalid_actions_seen()
