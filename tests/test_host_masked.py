"""Masked host-driven steps (BatchedEnvironment.step_host with `mask` / `episodes_left`, bsb_step_host_masked) on the
host path.

One masked host step must equal, bit for bit, `rollout(1, actions, mask=, episodes_left=)` on a twin handle: every
output entry written (unwritten ones keep a sentinel), steps_done, the budgets, bsuite_info(), episode statistics, log
rows and the raw state.  With budgets the mask is written back as `old_mask & (left > 0)`; without, it is only read.
`run_host_episodes` must equal `run_episodes` driven by the same actions."""
import ctypes

import numpy as np
import pytest
import torch

import bsuite_b200
from bsuite_b200 import _lib
from bsuite_b200 import analysis
from bsuite_b200 import rollouts
from bsuite_b200 import suite
from tests import test_masked as tm
from tests import test_masked_rollout as tr

SENTINEL = tm.SENTINEL
SCALARS = ('reward', 'discount', 'step_type')


def make_calls(batch, num_actions, seed, calls=40, densities=tm.DENSITIES):
  """[(mask bool [B], budgets int64 [B] or None, actions int32 [B])]: test_masked's plans (resets dropped), budgets of
  0 to 3 episodes on every other call; lanes whose mask is clear get out-of-range actions, which must never be read."""
  plan = tm.make_plan(batch, calls, num_actions, seed, densities=densities, reset_every=calls + 1)
  rng = np.random.default_rng(seed + 1)
  return [(mask, rng.integers(0, 4, batch).astype(np.int64) if c % 2 == 0 else None, actions)
          for c, (_, mask, actions) in enumerate(plan)]


def fill(buffers):
  for name in tm.FIELDS:
    tensor = getattr(buffers, name, None)
    if tensor is not None:
      tensor.fill_(SENTINEL)


def host_step(env, call, host, out, mask_dtype=torch.bool):
  """One masked host step of `call`; returns (mask after the call, budgets after it or None)."""
  mask, budgets, actions = call
  mask_t = torch.tensor(mask).to(mask_dtype)      # a copy: the call writes it back
  left = None if budgets is None else torch.tensor(budgets).to(env.device)
  fill(host)
  fill(out)
  env.step_host(torch.as_tensor(actions), host, out, mask=mask_t, episodes_left=left)
  return mask_t.bool().numpy(), None if left is None else left.cpu().numpy()


def twin_step(twin, call, out):
  """The same call as a one-step masked rollout; returns the budgets after it (or None)."""
  mask, budgets, actions = call
  left = None if budgets is None else torch.tensor(budgets).to(twin.device)
  fill(out)
  twin.rollout(1, actions=torch.as_tensor(actions)[None].to(twin.device), out=out,
               mask=torch.as_tensor(mask).to(twin.device), episodes_left=left)
  return None if left is None else left.cpu().numpy()


def check_calls(env, twin, calls, mask_dtype=torch.bool):
  host, out = env.make_host_buffers(), env.make_buffers()
  twin_out = twin.make_buffers(1)
  for c, call in enumerate(calls):
    mask_after, left = host_step(env, call, host, out, mask_dtype)
    twin_left = twin_step(twin, call, twin_out)
    for name in SCALARS:
      assert torch.equal(getattr(host, name).cpu(), getattr(twin_out, name)[0].cpu()), f'{name} at call {c}'
    assert torch.equal(out.observation.cpu(), twin_out.observation[0].cpu()), f'observation at call {c}'
    if left is None:
      assert twin_left is None
      assert np.array_equal(mask_after, call[0]), f'the mask of call {c} was written without budgets'
    else:
      assert np.array_equal(left, twin_left), f'budgets after call {c}'
      assert np.array_equal(mask_after, call[0] & (left > 0)), f'mask write-back of call {c}'
    assert env.steps_done == twin.steps_done == c + 1
  acc, acc_twin = tm.accumulators(env), tm.accumulators(twin)
  for key in acc_twin:
    assert torch.equal(acc[key], acc_twin[key]), key
  assert tr.raw_state(env) == tr.raw_state(twin)


@pytest.mark.parametrize('bsuite_id', suite.one_per_experiment())
def test_every_experiment_equals_a_one_step_masked_rollout(bsuite_id, request):
  tm._mnist_if_needed(bsuite_id, request)
  env, twin = tr.twins(bsuite_id, 9, lane_offset=3, record_rows=True)
  check_calls(env, twin, make_calls(env.batch, env.num_actions, seed=sum(map(ord, bsuite_id))))


@pytest.mark.parametrize('bsuite_id,kwargs', [
    ('catch/0', dict(autoreset='same_step')),
    ('deep_sea/2', dict(autoreset='same_step', obs_dtype='bfloat16')),
    ('cartpole/1', dict(autoreset='same_step')),
    ('catch/0', dict(rng='mt19937')),
    ('deep_sea_stochastic/1', dict(rng='mt19937')),
    ('cartpole_noise/3', dict(rng='mt19937')),
    ('deep_sea/0', dict(obs_dtype='uint8')),
    ('bandit_noise/1', dict(reward_dtype='float64')),
])
def test_handle_kinds_equal_a_one_step_masked_rollout(bsuite_id, kwargs):
  env, twin = tr.twins(bsuite_id, 7, seed=5, record_rows=not kwargs.get('rng'), **kwargs)
  check_calls(env, twin, make_calls(env.batch, env.num_actions, seed=len(bsuite_id), densities=(0.5, 1.0, 0.03, 0.7)))


@pytest.mark.parametrize('name,ragged', [('catch', False), ('bandit', False), ('cartpole_noise', False),
                                         ('deep_sea', True), ('memory_size', True), ('umbrella_distract', True)])
def test_packed_and_ragged_equal_a_one_step_masked_rollout(name, ragged):
  kw = dict(device='cpu', seed=4, track_episodes=True, record_rows=True, ragged=ragged)
  env, twin = bsuite_b200.load_experiment(name, 3, **kw), bsuite_b200.load_experiment(name, 3, **kw)
  check_calls(env, twin, make_calls(env.batch, env.num_actions, seed=len(name), calls=30))


def test_uint8_masks_and_empty_and_full_masks():
  env, twin = tr.twins('catch/0', 6)
  B, n = env.batch, env.num_actions
  calls = [(np.zeros(B, bool), np.full(B, 2, np.int64), np.full(B, n + 4, np.int32)),
           (np.ones(B, bool), None, np.arange(B, dtype=np.int32) % n)]
  calls += [(np.ones(B, bool), np.full(B, 1, np.int64), np.arange(B, dtype=np.int32) % n)] * 12
  check_calls(env, twin, calls, mask_dtype=torch.uint8)


def test_mask_write_back_is_in_place_and_only_with_budgets():
  env = bsuite_b200.load_from_id('catch/0', batch=4, device='cpu', seed=0)
  host, out = env.make_host_buffers(), env.make_buffers()
  mask = torch.tensor([True, True, False, True])
  left = torch.tensor([0, 1, 5, 2])
  for _ in range(40):      # catch: 9 steps per episode (rows - 1)
    env.step_host(torch.zeros(4, dtype=torch.int32), host, out, mask=mask, episodes_left=left)
  assert mask.tolist() == [False, False, False, False]
  assert left.tolist() == [0, 0, 5, 0]
  raw = torch.tensor([1, 0, 1, 1], dtype=torch.uint8)
  env.step_host(torch.zeros(4, dtype=torch.int32), host, out, mask=raw)
  assert raw.tolist() == [1, 0, 1, 1]
  view = torch.tensor([1, 1, 1, 1], dtype=torch.uint8)
  env.step_host(torch.zeros(4, dtype=torch.int32), host, out, mask=view, episodes_left=torch.tensor([0, 3, -1, 1]))
  assert view.tolist() == [0, 1, 0, 1]


def test_mask_arguments_are_checked():
  env = bsuite_b200.load_from_id('catch/0', batch=4, device='cpu', seed=0)
  host, out = env.make_host_buffers(), env.make_buffers()
  actions = torch.zeros(4, dtype=torch.int32)
  mask = torch.ones(4, dtype=torch.bool)
  for bad, match in ((torch.ones(4, dtype=torch.int32), 'bool or uint8'), (np.ones(4, bool), 'bool or uint8'),
                     (torch.ones(5, dtype=torch.bool), 'shape'), (torch.ones(8, dtype=torch.bool)[::2], 'contiguous'),
                     (torch.ones(4, dtype=torch.bool, device='meta'), 'host memory')):
    with pytest.raises(ValueError, match=match):
      env.step_host(actions, host, out, mask=bad)
  with pytest.raises(ValueError, match='needs mask'):
    env.step_host(actions, host, out, episodes_left=torch.ones(4, dtype=torch.int64))
  for bad, match in ((torch.ones(4, dtype=torch.int32), 'int64'), (torch.ones(5, dtype=torch.int64), 'shape'),
                     (torch.ones(4, dtype=torch.int64, device='meta'), 'live on'),
                     (torch.ones(8, dtype=torch.int64)[::2], 'contiguous')):
    with pytest.raises(ValueError, match=match):
      env.step_host(actions, host, out, mask=mask, episodes_left=bad)
  same = bsuite_b200.load_from_id('catch/0', batch=4, device='cpu', seed=0, autoreset='same_step')
  finals = same.make_host_buffers()
  finals.final_observation = same.make_buffers(final_observation=True).final_observation
  with pytest.raises(ValueError, match='final observations'):
    same.step_host(actions, finals, same.make_buffers(), mask=mask)
  assert env.steps_done == 0


def test_bad_action_of_an_active_lane_moves_nothing():
  env = bsuite_b200.load_from_id('bandit/0', batch=4, device='cpu', seed=2, track_episodes=True, record_rows=True)
  host, out = env.make_host_buffers(), env.make_buffers()
  env.step_host(torch.zeros(4, dtype=torch.int32), host, out, mask=torch.ones(4, dtype=torch.bool))
  n = env.num_actions
  mask = torch.tensor([True, False, True, True])
  left = torch.tensor([2, 2, 0, 2])
  fill(host)
  fill(out)
  # lane 1 is masked out and lane 2's budget is spent: their bad actions are never read
  env.step_host(torch.tensor([0, n + 3, -1, 1], dtype=torch.int32), host, out, mask=mask, episodes_left=left)
  assert mask.tolist() == [True, False, False, True] and env.steps_done == 2
  state = tr.raw_state(env)
  fill(host)
  fill(out)
  with pytest.raises(_lib.EngineError, match='active lane 3'):
    env.step_host(torch.tensor([0, 0, 0, n], dtype=torch.int32), host, out, mask=mask, episodes_left=left)
  assert tr.raw_state(env) == state and env.steps_done == 2
  assert mask.tolist() == [True, False, False, True] and left.tolist() == [1, 2, 0, 1]
  assert torch.all(host.reward == SENTINEL) and torch.all(out.observation == SENTINEL)


def stream_agent(env, action_seed):
  return tr.stream_agent(env, action_seed)


def host_policy(env, action_seed):
  def policy(call, timestep, observation, mask):
    del call, timestep, observation, mask
    return torch.as_tensor(env.random_actions(1, action_seed, first_step=env.steps_done)[0])
  return policy


@pytest.mark.parametrize('bsuite_id', suite.one_per_experiment())
def test_run_host_episodes_equals_run_episodes(bsuite_id, request):
  tm._mnist_if_needed(bsuite_id, request)
  env, twin = tr.twins(bsuite_id, 5, lane_offset=2, record_rows=True)
  calls = rollouts.run_host_episodes(host_policy(env, 3), env, 2)
  twin_calls = rollouts.run_episodes(stream_agent(twin, 3), twin, 2, check_every=1)
  assert calls == twin_calls
  acc, acc_twin = tm.accumulators(env), tm.accumulators(twin)
  for key in acc_twin:
    assert torch.equal(acc[key], acc_twin[key]), key
  assert torch.all(env.episode_stats()['episode'] == 2)


def test_run_host_episodes_uses_each_settings_budget_and_scores_equal():
  kw = dict(device='cpu', seed=1, track_episodes=True, record_rows=True)
  env, twin = bsuite_b200.load_experiment('bandit', 3, **kw), bsuite_b200.load_experiment('bandit', 3, **kw)
  specs = list(env._pack[1]) + [spec for spec in twin._pack[1] if all(spec is not s for s in env._pack[1])]
  budgets = [spec.bsuite_num_episodes for spec in specs]
  small = [3 + k % 4 for k in range(len(env._pack[1]))]
  for k, spec in enumerate(specs):             # a short run: each setting's budget lowered in place
    spec.bsuite_num_episodes = small[k % len(small)]
  try:
    seen = []

    def policy(call, timestep, observation, mask):
      seen.append(mask.clone())
      return host_policy(env, 7)(call, timestep, observation, mask)
    rollouts.run_host_episodes(policy, env)
    rollouts.run_episodes(stream_agent(twin, 7), twin)
  finally:
    for spec, n in zip(specs, budgets):
      spec.bsuite_num_episodes = n
  assert seen[0].all() and seen[-1].any() and seen[-1].sum() < env.batch
  assert env.episode_stats()['episode'].tolist() == [float(n) for n in small for _ in range(3)]
  acc, acc_twin = tm.accumulators(env), tm.accumulators(twin)
  for key in acc_twin:
    assert torch.equal(acc[key], acc_twin[key]), key
  a, b = analysis.bsuite_score(env), analysis.bsuite_score(twin)
  assert torch.equal(a.score.view(torch.int64), b.score.view(torch.int64))      # bit for bit, NaN for absent ones
  assert torch.equal(a.finished, b.finished)
  assert torch.equal(a.tag_score.view(torch.int64), b.tag_score.view(torch.int64))


def test_abi_statuses():
  lib = _lib.load()
  env = bsuite_b200.load_from_id('catch/0', batch=2, device='cpu', seed=0)
  host, out = env.make_host_buffers(), env.make_buffers()
  outputs = _lib.Outputs.from_buffer_copy(host.bind(env._obs_dtype))
  outputs.observation = out.observation.data_ptr()
  actions = torch.zeros(2, dtype=torch.int32)
  mask = torch.ones(2, dtype=torch.uint8)
  assert lib.bsb_step_host_masked(env._handle.ptr, actions.data_ptr(), None, None, ctypes.byref(outputs), None, None,
                                  0) == 1
  assert b'needs a mask' in lib.bsb_last_error()
  assert lib.bsb_step_host_masked(None, actions.data_ptr(), mask.data_ptr(), None, ctypes.byref(outputs), None, None,
                                  0) == 1
  fin = _lib.Outputs.from_buffer_copy(outputs)
  fin.final_observation = out.observation.data_ptr()
  assert lib.bsb_step_host_masked(env._handle.ptr, actions.data_ptr(), mask.data_ptr(), None, ctypes.byref(fin), None,
                                  None, 0) != 0
  assert b'final_observation' in lib.bsb_last_error()
  assert lib.bsb_step_host_masked(env._handle.ptr, actions.data_ptr(), mask.data_ptr(), None, ctypes.byref(outputs),
                                  None, None, 0) == 0
  assert env.steps_done == 1
