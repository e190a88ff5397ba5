"""Output-free masked rollouts (BatchedEnvironment.advance, bsb_advance_masked) on the host path, and a sweep run to its
episode budgets (SweepBatch.run_random_episodes).

`advance(T, action_seed, mask, episodes_left)` must equal `rollout(T, action_seed=..., out=..., mask=...,
episodes_left=...)` on a twin handle bit for bit in everything but the outputs: the budgets, steps_done,
bsuite_info(), episode statistics, log rows and the raw state.  umbrella_chain draws its distractors while it renders
an observation, so its cases show that the draws are still made when nothing is rendered."""
import ctypes

import numpy as np
import pytest
import torch

import bsuite_b200
from bsuite_b200 import _lib
from bsuite_b200 import analysis
from bsuite_b200 import build as bsb_build
from bsuite_b200 import rollouts
from bsuite_b200 import suite
from bsuite_b200 import sweep
from tests import test_masked as tm
from tests import test_masked_rollout as tr


def as_tensors(env, launch):
  """(T, mask, budgets or None) of a make_launches entry as tensors on the environment's device (fresh budgets)."""
  T, mask, budgets, _ = launch
  left = None if budgets is None else torch.tensor(budgets).to(env.device)
  return T, torch.as_tensor(mask).to(env.device), left


def check_advance_launches(env, twin, launches, action_seed=5):
  """Runs every launch as `advance` on `env` and as a masked rollout (sampled actions, full outputs) on `twin`, and
  compares the two after each launch."""
  for k, launch in enumerate(launches):
    T, mask, left = as_tensors(env, launch)
    _, twin_mask, twin_left = as_tensors(twin, launch)
    env.advance(T, action_seed=action_seed, mask=mask, episodes_left=left)
    twin.rollout(T, action_seed=action_seed, out=twin.make_buffers(T, with_actions=True,
                                                                    final_observation=twin._autoreset == 'same_step'),
                 mask=twin_mask, episodes_left=twin_left)
    if left is not None:
      assert torch.equal(left.cpu(), twin_left.cpu()), f'budgets after launch {k}'
    assert env.steps_done == twin.steps_done
    acc, acc_twin = tm.accumulators(env), tm.accumulators(twin)
    for key in acc_twin:
      assert torch.equal(acc[key], acc_twin[key]), f'{key} after launch {k}'
    assert tr.raw_state(env) == tr.raw_state(twin), f'state after launch {k}'


def launches_for(env, seed):
  return tr.make_launches(env.batch, env.num_actions, seed=seed, densities=(1.0, 0.0, 0.5, 0.03, 1.0, 0.5, 0.7),
                          steps=(5, 3, 9, 1, 16, 7, 64))


@pytest.mark.parametrize('bsuite_id', suite.one_per_experiment())
def test_every_experiment_equals_masked_rollouts(bsuite_id, request):
  tm._mnist_if_needed(bsuite_id, request)
  env, twin = tr.twins(bsuite_id, 37, lane_offset=3, record_rows=True)
  check_advance_launches(env, twin, launches_for(env, seed=sum(map(ord, bsuite_id))))


@pytest.mark.parametrize('bsuite_id,kwargs', [
    ('catch/0', dict(autoreset='same_step')),
    ('umbrella_distract/3', dict(autoreset='same_step')),
    ('deep_sea/2', dict(obs_dtype='bfloat16')),
    ('umbrella_distract/9', dict(obs_dtype='bfloat16')),
    ('catch/0', dict(rng='mt19937')),
    ('umbrella_distract/5', dict(rng='mt19937')),
    ('cartpole_noise/3', {}),
    ('bandit_noise/1', dict(reward_dtype='float64')),
])
def test_handle_kinds_equal_masked_rollouts(bsuite_id, kwargs):
  env, twin = tr.twins(bsuite_id, 35, record_rows=not kwargs.get('rng'), **kwargs)
  check_advance_launches(env, twin, launches_for(env, seed=len(bsuite_id) + 1))


@pytest.mark.parametrize('name,ragged', [('catch_noise', False), ('umbrella_distract', True), ('deep_sea', True)])
def test_packed_and_ragged_equal_masked_rollouts(name, ragged):
  kw = dict(device='cpu', seed=4, track_episodes=True, record_rows=True, ragged=ragged)
  env, twin = bsuite_b200.load_experiment(name, 5, **kw), bsuite_b200.load_experiment(name, 5, **kw)
  check_advance_launches(env, twin, launches_for(env, seed=len(name)))


def test_mask_none_is_every_lane():
  env, twin = tr.twins('catch/1', 33, record_rows=True)
  left, twin_left = torch.full((33,), 2, dtype=torch.int64), torch.full((33,), 2, dtype=torch.int64)
  for T in (3, 20, 7):
    env.advance(T, action_seed=4, episodes_left=left)
    twin.advance(T, action_seed=4, mask=torch.ones(33, dtype=torch.uint8), episodes_left=twin_left)
  assert torch.equal(left, twin_left) and env.steps_done == twin.steps_done == 30
  assert tr.raw_state(env) == tr.raw_state(twin)


def old_run_random_episodes(env, num_episodes=None, action_seed=0, steps_per_launch=64):
  """rollouts.run_random_episodes as it was before `advance`: masked rollouts that write every output."""
  T = int(steps_per_launch)
  left = rollouts.episode_budget(env, num_episodes)
  mask = left > 0
  env.reset(out=env.make_buffers(), mask=mask)
  out = env.make_buffers(T)
  calls = 0
  while bool((left > 0).any()):
    env.rollout(T, action_seed=action_seed, out=out, mask=mask, episodes_left=left)
    calls += T
  return calls


@pytest.mark.parametrize('make', [
    lambda: bsuite_b200.load_experiment('umbrella_distract', 3, device='cpu', seed=5, track_episodes=True,
                                        record_rows=True, ragged=True),
    lambda: bsuite_b200.load_from_id('catch/2', batch=9, device='cpu', seed=5, track_episodes=True, record_rows=True),
    lambda: bsuite_b200.load_from_id('bandit/0', batch=9, device='cpu', seed=5, track_episodes=True, record_rows=True,
                                     autoreset='same_step'),
], ids=['umbrella_distract-ragged', 'catch', 'bandit-same_step'])
def test_launch_length_does_not_matter(make):
  """A lane is active at every call from the reset until its budget is spent, so its j-th step takes the action of
  global index s0 + j whatever the launch length: accumulators, log rows and scores agree at 7 and 64 calls per
  launch, and with the output-writing rollouts of before."""
  a, b, c = make(), make(), make()
  calls_a = rollouts.run_random_episodes(a, 3, action_seed=2, steps_per_launch=7)
  calls_b = rollouts.run_random_episodes(b, 3, action_seed=2, steps_per_launch=64)
  calls_c = old_run_random_episodes(c, 3, action_seed=2, steps_per_launch=64)
  assert calls_a % 7 == 0 and calls_b == calls_c
  acc = tm.accumulators(a)
  for other in (b, c):
    acc_other = tm.accumulators(other)
    for key in acc:
      assert torch.equal(acc[key], acc_other[key]), key
  assert torch.all(a.episode_stats()['episode'] == 3)
  assert b.steps_done == c.steps_done
  scores = [analysis.bsuite_score(env) for env in (a, b, c)]
  for other in scores[1:]:
    assert torch.equal(scores[0].score.view(torch.int64), other.score.view(torch.int64))


# ----- a whole sweep to its budgets -----------------------------------------------------------------------------------
IDS = list(sweep.SWEEP)


def id_rows(batch, bsuite_id):
  """(counts [L], [rows [count, n_cols] of each lane]) of `bsuite_id`'s lanes in a SweepBatch."""
  if batch.packed:
    env = batch.pack_of(bsuite_id)
    lanes = env.lanes_of(bsuite_id)
  else:
    env, lanes = batch.envs[bsuite_id], slice(None)
  rows = env.logged_rows()
  counts, block = rows['counts'][lanes].cpu(), rows['rows'][..., lanes].cpu()
  return counts, [block[:int(n), :, j] for j, n in enumerate(counts)]


def assert_same_sweeps(a, b, ids=tuple(IDS)):
  assert torch.equal(a.local_returns(), b.local_returns())
  for i in ids:
    (counts_a, rows_a), (counts_b, rows_b) = id_rows(a, i), id_rows(b, i)
    assert torch.equal(counts_a, counts_b), i
    for x, y in zip(rows_a, rows_b):
      assert torch.equal(x, y), i
  sa, sb = analysis.bsuite_score(a), analysis.bsuite_score(b)
  for x, y in ((sa.score, sb.score), (sa.tag_score, sb.tag_score)):
    assert torch.equal(x.view(torch.int64), y.view(torch.int64))
  assert torch.equal(sa.finished, sb.finished)


@pytest.fixture(scope='module')
def sweeps(mnist_dir):
  """The full 468-id sweep at 3 lanes, 2 episodes per lane: packed, one handle per id, and packs driven one by one
  with output-writing masked rollouts."""
  del mnist_dir
  kw = dict(lanes=3, device='cpu', seed=8, record_rows=True)
  packed, plain, driven = (suite.SweepBatch(IDS, packed=p, **kw) for p in (True, False, True))
  calls = packed.run_random_episodes(num_episodes=2, action_seed=3)
  plain_calls = plain.run_random_episodes(num_episodes=2, action_seed=3)
  driven_calls = {k: old_run_random_episodes(env, 2, action_seed=3, steps_per_launch=suite.RUN_STEPS_PER_LAUNCH)
                  for k, env in driven.envs.items()}
  yield packed, plain, driven, calls, plain_calls, driven_calls
  for batch in (packed, plain, driven):
    batch.close()


def test_sweep_packed_equals_one_handle_per_id(sweeps):
  packed, plain, _, calls, plain_calls, _ = sweeps
  assert list(calls) == list(packed.envs) and list(plain_calls) == IDS
  assert all(n % suite.RUN_STEPS_PER_LAUNCH == 0 and n > 0 for n in list(calls.values()) + list(plain_calls.values()))
  assert_same_sweeps(packed, plain)
  assert torch.all(packed.local_returns()[:, 1] == 2 * 3)        # every id: 2 episodes on each of 3 lanes
  assert analysis.bsuite_score(packed).score.isfinite().any()


def test_sweep_equals_packs_driven_with_masked_rollouts(sweeps):
  packed, _, driven, calls, _, driven_calls = sweeps
  assert calls == driven_calls
  assert_same_sweeps(packed, driven)
  for k, env in packed.envs.items():
    assert tr.raw_state(env) == tr.raw_state(driven.envs[k]), k


def by_setting(acc, env):
  """{key: [per-setting [..., L] tensors]} of a pack's accumulators."""
  lanes = env.lanes_per_setting
  return {key: [value[..., s * lanes:(s + 1) * lanes] for s in range(len(env.bsuite_ids))] for key, value in acc.items()}


def test_sweep_two_ranks_equal_world_one(sweeps):
  """Rank r of world 2 holds lanes [r*L/2, (r+1)*L/2) of every setting: put together, each setting's lanes equal
  world 1's, accumulators and log rows included."""
  packed = sweeps[0]
  ranks = [suite.SweepBatch(IDS, lanes=3, device='cpu', seed=8, record_rows=True, packed=True, rank=r, world=2)
           for r in range(2)]
  for rank in ranks:
    rank.run_random_episodes(num_episodes=2, action_seed=3)
  for k, env in packed.envs.items():
    want = by_setting(tm.accumulators(env), env)
    parts = [by_setting(tm.accumulators(rank.envs[k]), rank.envs[k]) for rank in ranks]
    for key, settings in want.items():
      for s, value in enumerate(settings):
        assert torch.equal(torch.cat([part[key][s] for part in parts], dim=-1), value), (k, key, s)
  for rank in ranks:
    rank.close()


def test_sweep_with_no_budget_makes_no_launch():
  batch = suite.SweepBatch(['catch/0', 'bandit/3'], lanes=4, device='cpu', seed=1, packed=True)
  steps = {k: env.steps_done for k, env in batch.envs.items()}
  assert batch.run_random_episodes(num_episodes=0) == {k: 0 for k in batch.envs}
  assert {k: env.steps_done for k, env in batch.envs.items()} == {k: n + 1 for k, n in steps.items()}
  with pytest.raises(ValueError, match='steps_per_launch'):
    batch.run_random_episodes(steps_per_launch=0)
  batch.close()


# ----- arguments --------------------------------------------------------------------------------------------------
def test_advance_arguments_are_checked():
  env = bsuite_b200.load_from_id('catch/0', batch=4, device='cpu', seed=0)
  ones = torch.ones(4, dtype=torch.bool)
  with pytest.raises(ValueError, match='shape'):
    env.advance(3, mask=torch.ones(5, dtype=torch.bool))
  with pytest.raises(ValueError, match='bool or uint8'):
    env.advance(3, mask=torch.ones(4, dtype=torch.int32))
  with pytest.raises(ValueError, match='int64'):
    env.advance(3, mask=ones, episodes_left=torch.ones(4, dtype=torch.int32))
  with pytest.raises(ValueError, match='int64'):
    env.advance(3, mask=ones, episodes_left=[1, 1, 1, 1])
  with pytest.raises(ValueError, match='shape'):
    env.advance(3, mask=ones, episodes_left=torch.ones(5, dtype=torch.int64))
  with pytest.raises(ValueError, match='contiguous'):
    env.advance(3, mask=ones, episodes_left=torch.ones(8, dtype=torch.int64)[::2])
  for T in (0, -2):
    with pytest.raises(_lib.EngineError, match='num_steps'):
      env.advance(T, mask=ones)
  assert env.steps_done == 0
  env.advance(3, mask=ones)
  assert env.steps_done == 3


def test_abi_statuses():
  lib = _lib.load()
  assert lib.bsb_abi_version() == 15
  cfg = _lib.Config()
  cfg.family, cfg.rows, cfg.columns, cfg.reward_scale = _lib.CATCH, 10, 5, 1.0
  handle = ctypes.c_void_p()
  _lib.check(lib.bsb_create(ctypes.byref(cfg), 3, _lib.DEVICE_HOST, 5, 0, ctypes.byref(handle)))
  mask = np.array([1, 0, 1], np.uint8)
  left = np.array([2, 2, 0], np.int64)
  advance = lib.bsb_advance_masked
  assert advance(None, 4, 0, mask.ctypes.data, None, None) == 1
  assert advance(handle, 4, 0, None, None, None) == 1
  assert b'mask' in lib.bsb_last_error()
  assert advance(handle, 0, 0, mask.ctypes.data, None, None) == 1
  assert advance(handle, -2, 0, mask.ctypes.data, None, None) == 1
  assert b'num_steps' in lib.bsb_last_error()
  steps = ctypes.c_int64()
  _lib.check(lib.bsb_steps_done(handle, ctypes.byref(steps)))
  assert steps.value == 0
  _lib.check(advance(handle, 4, 3, mask.ctypes.data, left.ctypes.data, None))
  _lib.check(advance(handle, 4, 3, mask.ctypes.data, None, None))
  _lib.check(lib.bsb_steps_done(handle, ctypes.byref(steps)))
  assert steps.value == 8
  assert left.tolist() == [2, 2, 0]              # catch episodes are longer than 4 steps: no LAST yet
  _lib.check(lib.bsb_destroy(handle))


# ----- the GPU cases cover the list -------------------------------------------------------------------------------
def test_gpu_cases_cover_every_masked_kernel_of_the_list():
  """Every variant of the list, times its bit sources, has a case in test_advance_gpu.py: with it the CALL_ADVANCE
  instantiation of masked_kernel."""
  from tests import test_advance_gpu as g
  want = {(family, obs, mode, 'philox') for variants in bsb_build.variant_list().values()
          for family, obs, mode, _, _ in variants}
  want |= {(family, obs, mode, 'mt19937') for variants in bsb_build.variant_list().values()
           for family, obs, mode, mt, _ in variants if mt}
  assert len(want) == sum(1 + int(mt) for variants in bsb_build.variant_list().values() for *_, mt, _ in variants)
  assert set(g.CASES) == want
