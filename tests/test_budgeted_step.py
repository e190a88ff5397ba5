"""Budgeted steps (BatchedEnvironment.step with `episodes_left` / `previous`, bsb_step_budgeted) on the host path, the
agent loop built on them (rollouts.run_episodes) and whole-sweep agent loops (SweepBatch.run_episodes).

A budgeted step must equal, bit for bit, its model on a twin handle: copy out -> previous where the mask is set, then
a one-step masked rollout with the same mask and budgets, then mask &= (budget before the call > 0).  Compared are
out, previous, mask, budgets, steps_done, bsuite_info(), episode statistics, log rows and the raw state.
`run_episodes` must show an agent exactly what the loop it replaced showed (kept here as `parent_run_episodes`)."""
import ctypes

import numpy as np
import pytest
import torch

import bsuite_b200
from bsuite_b200 import _lib
from bsuite_b200 import analysis
from bsuite_b200 import rollouts
from bsuite_b200 import suite
from tests import test_advance as ta
from tests import test_masked as tm
from tests import test_masked_rollout as tr

OUT_FIELDS = ('observation', 'reward', 'discount', 'step_type', 'final_observation')


# ----- the model ------------------------------------------------------------------------------------------------------
def obs_parts(env, tensor):
  """Per-setting [L, ...] views of an observation tensor [B, ...] (a ragged pack's flat buffer included)."""
  return env.split_observation(tensor)


def model_step(twin, actions, mask, left, out, previous):
  """The budgeted step's model on `twin`: `out` is a make_buffers(1) set (leading T axis), `previous` a step set;
  `mask` (uint8) and `left` are updated in place like the call's."""
  m = mask.bool()
  for name in OUT_FIELDS:
    src, dst = getattr(out, name), getattr(previous, name)
    if src is None or dst is None:
      continue
    if name == 'observation':
      lanes = twin.lanes_per_setting
      for k, (s, d) in enumerate(zip(obs_parts(twin, src[0]), obs_parts(twin, dst))):
        sel = m[k * lanes:(k + 1) * lanes]
        d[sel] = s[sel]
    else:
      dst[m] = src[0][m]
  before = left.clone()
  twin.rollout(1, actions=actions.unsqueeze(0), out=out, mask=mask, episodes_left=left)
  mask &= (before > 0).to(mask.dtype)


def make_pair(env):
  """(out, previous) of a budgeted step and the twin's (out [1, ...], previous), filled alike."""
  final = env.autoreset == 'same_step'
  return env.make_buffers(final_observation=final), env.make_buffers(final_observation=final)


def fill_like(bufs, twin_bufs, seed):
  """Fills both sets with the same random contents (twin_bufs[0] has a leading T = 1 axis)."""
  g = torch.Generator().manual_seed(seed)
  for (a, b) in zip(bufs, twin_bufs):
    for name in OUT_FIELDS:
      x, y = getattr(a, name), getattr(b, name)
      if x is None:
        continue
      v = torch.randint(0, 3, tuple(x.shape), generator=g).to(x.dtype).to(x.device)
      x.copy_(v)
      y.copy_(v.reshape(y.shape))


def assert_same_buffers(a, b, where, lead=False):
  for name in OUT_FIELDS:
    x, y = getattr(a, name), getattr(b, name)
    if x is None:
      assert y is None
      continue
    y = y[0] if lead else y
    assert torch.equal(x.cpu().view(torch.uint8) if x.dtype == torch.bfloat16 else x.cpu(),
                       y.cpu().view(torch.uint8) if y.dtype == torch.bfloat16 else y.cpu()), f'{name} {where}'


def assert_same_lanes(env, twin, where):
  assert env.steps_done == twin.steps_done, where
  acc, acc_twin = tm.accumulators(env), tm.accumulators(twin)
  for key in acc_twin:
    assert torch.equal(acc[key], acc_twin[key]), f'{key} {where}'
  assert tr.raw_state(env) == tr.raw_state(twin), f'state {where}'


def drive_against_model(env, twin, seed, min_calls=12, max_calls=4000, every=1, host=None):
  """Budgeted steps on `env` and their model on `twin`, from one masked reset, with random masks and budgets of 0-3
  episodes.  Every few calls some lanes are masked in again, so lanes whose budget is spent sit out (and have their
  mask cleared) more than once.  Runs until every lane has spent its budget and sat out at least twice.  `host` (a
  host-path handle like `env`): makes the same budgeted steps, and its masks and budgets must equal env's."""
  rng = np.random.default_rng(seed)
  B, dev = env.batch, env.device
  left = torch.as_tensor(rng.integers(0, 4, B).astype(np.int64)).to(dev)
  mask = torch.as_tensor(rng.random(B) < 0.8).to(dev).to(torch.uint8)
  twin_left, twin_mask = left.clone(), mask.clone()
  out, previous = make_pair(env)
  if host is not None:
    host_left, host_mask = left.cpu(), mask.cpu()
    host_out, host_prev = make_pair(host)
    host.reset(out=host_out, mask=torch.ones(B, dtype=torch.uint8))
  twin_out = twin.make_buffers(1, final_observation=env.autoreset == 'same_step')
  twin_prev = twin.make_buffers(final_observation=env.autoreset == 'same_step')
  fill_like((out, previous), (twin_out, twin_prev), seed)
  start = torch.ones(B, dtype=torch.uint8, device=dev)
  env.reset(out=out, mask=start)
  twin_reset = twin.make_buffers()
  for name in ('observation', 'reward', 'discount', 'step_type'):      # a ragged pack's gaps are never written
    getattr(twin_reset, name).copy_(getattr(twin_out, name)[0])
  twin.reset(out=twin_reset, mask=start)       # the twin's reset, moved into its T = 1 set
  for name in ('observation', 'reward', 'discount', 'step_type'):
    getattr(twin_out, name)[0].copy_(getattr(twin_reset, name))
  sat_out = torch.zeros(B, dtype=torch.int64)
  calls = 0
  assert_same_buffers(out, twin_out, 'after the reset', lead=True)
  while calls < max_calls:
    if calls >= min_calls and bool((left == 0).all()) and bool((sat_out >= 2).all()):
      break
    if calls % 9 == 8:                        # mask some lanes in again: spent ones sit out once more
      extra = torch.as_tensor(rng.random(B) < 0.5).to(dev).to(torch.uint8)
      mask |= extra
      twin_mask |= extra
      if host is not None:
        host_mask |= extra.cpu()
    actions = torch.as_tensor(rng.integers(0, env.num_actions, B).astype(np.int32)).to(dev)
    spent = ((mask != 0) & (left <= 0)).cpu()
    env.step(actions, out=out, mask=mask, episodes_left=left, previous=previous)
    model_step(twin, actions, twin_mask, twin_left, twin_out, twin_prev)
    if host is not None:
      host.step(actions.cpu(), out=host_out, mask=host_mask, episodes_left=host_left, previous=host_prev)
      assert torch.equal(mask.cpu(), host_mask) and torch.equal(left.cpu(), host_left), f'host path at call {calls}'
    calls += 1
    sat_out += spent.to(torch.int64)
    where = f'after call {calls}'
    assert torch.equal(mask, twin_mask), f'mask {where}'
    assert torch.equal(left, twin_left), f'budgets {where}'
    assert_same_buffers(out, twin_out, where, lead=True)
    assert_same_buffers(previous, twin_prev, f'previous {where}')
    if calls % every == 0:
      assert_same_lanes(env, twin, where)
  assert bool((left == 0).all()) and bool((sat_out >= 2).all()), 'the run ended before every lane sat out twice'
  assert_same_lanes(env, twin, 'at the end')
  return calls


@pytest.mark.parametrize('bsuite_id', suite.one_per_experiment())
def test_every_experiment_equals_the_model(bsuite_id, request):
  tm._mnist_if_needed(bsuite_id, request)
  env, twin = tr.twins(bsuite_id, 37, lane_offset=3, record_rows=True)
  drive_against_model(env, twin, seed=sum(map(ord, bsuite_id)), every=7)


@pytest.mark.parametrize('bsuite_id,kwargs', [
    ('catch/0', dict(rng='mt19937')),
    ('umbrella_distract/5', dict(rng='mt19937')),
    ('catch/0', dict(autoreset='same_step')),
    ('umbrella_distract/3', dict(autoreset='same_step')),
    ('bandit/0', dict(autoreset='same_step')),
    ('deep_sea/2', dict(obs_dtype='bfloat16')),
    ('umbrella_distract/9', dict(obs_dtype='bfloat16')),
    ('catch/1', dict(obs_dtype='uint8')),
    ('deep_sea/3', dict(obs_dtype='uint8')),
    ('bandit_noise/1', dict(reward_dtype='float64')),
])
def test_handle_kinds_equal_the_model(bsuite_id, kwargs):
  env, twin = tr.twins(bsuite_id, 35, record_rows=not kwargs.get('rng'), **kwargs)
  drive_against_model(env, twin, seed=len(bsuite_id) + 1)


def test_same_step_without_final_observations_equals_the_model():
  env, twin = tr.twins('catch/2', 33, record_rows=True, autoreset='same_step')
  rng = np.random.default_rng(5)
  B = env.batch
  left = torch.as_tensor(rng.integers(0, 4, B).astype(np.int64))
  mask = torch.ones(B, dtype=torch.uint8)
  twin_left, twin_mask = left.clone(), mask.clone()
  out, previous = env.make_buffers(), env.make_buffers()
  twin_out, twin_prev = twin.make_buffers(1), twin.make_buffers()
  fill_like((out, previous), (twin_out, twin_prev), 5)
  env.reset(out=out, mask=mask)
  twin_reset = twin.make_buffers()
  twin.reset(out=twin_reset, mask=twin_mask)
  for name in ('observation', 'reward', 'discount', 'step_type'):
    getattr(twin_out, name)[0].copy_(getattr(twin_reset, name))
  for call in range(60):
    actions = torch.as_tensor(rng.integers(0, env.num_actions, B).astype(np.int32))
    env.step(actions, out=out, mask=mask, episodes_left=left, previous=previous)
    model_step(twin, actions, twin_mask, twin_left, twin_out, twin_prev)
    assert torch.equal(mask, twin_mask) and torch.equal(left, twin_left), call
    assert_same_buffers(out, twin_out, call, lead=True)
    assert_same_buffers(previous, twin_prev, call)
  assert not bool(mask.any())
  assert_same_lanes(env, twin, 'at the end')


@pytest.mark.parametrize('name,ragged', [('catch_noise', False), ('bandit', False), ('umbrella_distract', True),
                                         ('deep_sea', True), ('memory_len', True)])
def test_packed_and_ragged_equal_the_model(name, ragged):
  kw = dict(device='cpu', seed=4, track_episodes=True, record_rows=True, ragged=ragged)
  env, twin = bsuite_b200.load_experiment(name, 5, **kw), bsuite_b200.load_experiment(name, 5, **kw)
  drive_against_model(env, twin, seed=len(name), every=5)


# ----- the agent's view -------------------------------------------------------------------------------------------
def parent_run_episodes(agent, environment, num_episodes=None, check_every=16):
  """rollouts.run_episodes as it was before budgeted steps: copies into a spare buffer set, LAST counts in torch."""
  B, device = environment.batch, environment.device
  budget = rollouts.episode_budget(environment, num_episodes)
  finished = torch.zeros(B, dtype=torch.int64, device=device)
  active = budget > 0
  out = environment.make_buffers()
  timestep = environment.reset(out=out, mask=active)
  spare = environment.make_buffers()
  calls = 0
  while True:
    if calls % max(int(check_every), 1) == 0 and not bool(active.any()):
      return calls
    actions = agent.select_action(timestep)
    spare.observation.copy_(out.observation)
    spare.reward.copy_(out.reward)
    spare.discount.copy_(out.discount)
    spare.step_type.copy_(out.step_type)
    previous = spare.timestep()
    new_timestep = environment.step(actions, out=out, mask=active)
    calls += 1
    agent.update(previous, actions, new_timestep)
    finished += ((new_timestep.step_type == 2) & active).to(torch.int64)
    active = finished < budget
    timestep = new_timestep


class RecordingAgent:
  """Random actions from its own numpy stream; records every value it is passed (as CPU copies)."""

  def __init__(self, env, seed):
    self.env, self.rng, self.seen, self.updates = env, np.random.default_rng(seed), [], []

  def _copy(self, timestep):
    """CPU copies of the four fields (a ragged pack's observation without the gaps between settings, which no call
    writes)."""
    obs = torch.cat([part.reshape(-1) for part in self.env.split_observation(timestep.observation)])
    return tuple(getattr(timestep, f).cpu().clone() for f in ('step_type', 'reward', 'discount')) + (obs.cpu(),)

  def select_action(self, timestep):
    self.seen.append(self._copy(timestep))
    return torch.as_tensor(self.rng.integers(0, self.env.num_actions, self.env.batch).astype(np.int32)).to(self.env.device)

  def update(self, timestep, actions, new_timestep):
    self.updates.append((self._copy(timestep), actions.cpu().clone(), self._copy(new_timestep)))


def assert_same_records(a, b):
  assert len(a.seen) == len(b.seen) and len(a.updates) == len(b.updates)

  def same(x, y):
    return torch.equal(x.view(torch.uint8) if x.dtype == torch.bfloat16 else x,
                       y.view(torch.uint8) if y.dtype == torch.bfloat16 else y)
  for c, (x, y) in enumerate(zip(a.seen, b.seen)):
    assert all(same(p, q) for p, q in zip(x, y)), f'select_action at call {c}'
  for c, ((t0, a0, n0), (t1, a1, n1)) in enumerate(zip(a.updates, b.updates)):
    assert torch.equal(a0, a1), f'actions at call {c}'
    assert all(same(p, q) for p, q in zip(t0, t1)), f'update timestep at call {c}'
    assert all(same(p, q) for p, q in zip(n0, n1)), f'update new_timestep at call {c}'


@pytest.mark.parametrize('check_every', [1, 5])
@pytest.mark.parametrize('bsuite_id,kwargs', [
    ('catch/0', {}),
    ('deep_sea/1', {}),
    ('umbrella_distract/2', {}),
    ('catch/1', dict(autoreset='same_step')),
    ('bandit/2', dict(autoreset='same_step')),
    ('memory_len/3', dict(autoreset='same_step')),
])
def test_run_episodes_shows_the_agent_what_the_parent_loop_showed(bsuite_id, kwargs, check_every):
  """On a same-step handle a merged LAST counts against the budget like any LAST."""
  env, twin = tr.twins(bsuite_id, 21, record_rows=True, **kwargs)
  agent, twin_agent = RecordingAgent(env, 3), RecordingAgent(twin, 3)
  calls = rollouts.run_episodes(agent, env, num_episodes=3, check_every=check_every)
  twin_calls = parent_run_episodes(twin_agent, twin, num_episodes=3, check_every=check_every)
  assert calls == twin_calls and calls % check_every == 0
  assert_same_records(agent, twin_agent)
  assert torch.all(env.episode_stats()['episode'] == 3)
  acc, acc_twin = tm.accumulators(env), tm.accumulators(twin)
  for key in acc_twin:
    assert torch.equal(acc[key], acc_twin[key]), key


def test_run_episodes_on_a_ragged_pack_shows_the_agent_what_the_parent_loop_showed():
  kw = dict(device='cpu', seed=6, track_episodes=True, record_rows=True, ragged=True)
  env, twin = (bsuite_b200.load_experiment('deep_sea', 4, settings=[0, 3, 7], **kw) for _ in range(2))
  agent, twin_agent = RecordingAgent(env, 8), RecordingAgent(twin, 8)
  assert rollouts.run_episodes(agent, env, num_episodes=2) == parent_run_episodes(twin_agent, twin, num_episodes=2)
  assert_same_records(agent, twin_agent)


# ----- whole-sweep agent loops ------------------------------------------------------------------------------------
IDS = ['catch/0', 'catch/4', 'deep_sea/0', 'deep_sea/3', 'umbrella_distract/1', 'umbrella_distract/6', 'bandit/2',
       'bandit_noise/0', 'memory_len/0', 'memory_len/5', 'discounting_chain/1', 'cartpole_noise/2']


def recording_agents(batch, seed=3):
  return {k: RecordingAgent(env, seed + i) for i, (k, env) in enumerate(batch.envs.items())}


def sweep_rows(batch, ids):
  return [ta.id_rows(batch, i) for i in ids]


def assert_same_sweep_results(a, b, ids=tuple(IDS)):
  assert torch.equal(a.local_returns(), b.local_returns())
  for i in ids:
    (ca, ra), (cb, rb) = ta.id_rows(a, i), ta.id_rows(b, i)
    assert torch.equal(ca, cb), i
    for x, y in zip(ra, rb):
      assert torch.equal(x, y), i
  sa, sb = analysis.bsuite_score(a), analysis.bsuite_score(b)
  for x, y in ((sa.score, sb.score), (sa.tag_score, sb.tag_score)):
    assert torch.equal(x.view(torch.int64), y.view(torch.int64))


@pytest.mark.parametrize('packed', [True, False])
def test_sweep_run_episodes_equals_standalone_run_episodes(packed):
  kw = dict(lanes=3, device='cpu', seed=8, record_rows=True, packed=packed)
  batch, driven = suite.SweepBatch(IDS, **kw), suite.SweepBatch(IDS, **kw)
  agents, driven_agents = recording_agents(batch), recording_agents(driven)
  calls = batch.run_episodes(agents, num_episodes=2, check_every=4)
  driven_calls = {k: rollouts.run_episodes(driven_agents[k], env, num_episodes=2, check_every=4)
                  for k, env in driven.envs.items()}
  assert calls == driven_calls and list(calls) == list(batch.envs)
  for k in batch.envs:
    assert_same_records(agents[k], driven_agents[k])
    acc, acc_driven = tm.accumulators(batch.envs[k]), tm.accumulators(driven.envs[k])
    for key in acc_driven:
      assert torch.equal(acc[key], acc_driven[key]), (k, key)
    assert tr.raw_state(batch.envs[k]) == tr.raw_state(driven.envs[k]), k
  assert_same_sweep_results(batch, driven)
  assert torch.all(batch.local_returns()[:, 1] == 2 * 3)
  batch.close()
  driven.close()


def stream_agents(batch, action_seed):
  return {k: tr.stream_agent(env, action_seed) for k, env in batch.envs.items()}


@pytest.fixture(scope='module')
def stream_sweeps():
  """The IDS sweep at 4 lanes, 2 episodes per lane, played by the on-device action stream: packed and per id
  through run_episodes, and packed through run_random_episodes."""
  kw = dict(lanes=4, device='cpu', seed=5, record_rows=True)
  packed, plain, random_run = (suite.SweepBatch(IDS, packed=p, **kw) for p in (True, False, True))
  packed.run_episodes(stream_agents(packed, 9), num_episodes=2)
  plain.run_episodes(stream_agents(plain, 9), num_episodes=2)
  random_run.run_random_episodes(num_episodes=2, action_seed=9)
  yield packed, plain, random_run
  for batch in (packed, plain, random_run):
    batch.close()


def test_sweep_packed_equals_one_handle_per_id(stream_sweeps):
  packed, plain, _ = stream_sweeps
  assert_same_sweep_results(packed, plain)


def test_sweep_with_the_stream_agent_equals_run_random_episodes(stream_sweeps):
  """Everything but steps_done: run_random_episodes launches 1 024 calls at a time."""
  packed, _, random_run = stream_sweeps
  assert_same_sweep_results(packed, random_run)
  for k, env in packed.envs.items():
    acc, acc_random = tm.accumulators(env), tm.accumulators(random_run.envs[k])
    for key in acc_random:
      assert torch.equal(acc[key], acc_random[key]), (k, key)


def test_sweep_two_ranks_equal_world_one(stream_sweeps):
  packed = stream_sweeps[0]
  ranks = [suite.SweepBatch(IDS, lanes=4, device='cpu', seed=5, record_rows=True, packed=True, rank=r, world=2)
           for r in range(2)]
  for rank in ranks:
    rank.run_episodes(stream_agents(rank, 9), num_episodes=2)
  for k, env in packed.envs.items():
    want = ta.by_setting(tm.accumulators(env), env)
    parts = [ta.by_setting(tm.accumulators(rank.envs[k]), rank.envs[k]) for rank in ranks]
    for key, settings in want.items():
      for s, value in enumerate(settings):
        assert torch.equal(torch.cat([part[key][s] for part in parts], dim=-1), value), (k, key, s)
  for rank in ranks:
    rank.close()


def test_sweep_agent_loops_check_their_arguments():
  batch = suite.SweepBatch(['catch/0', 'bandit/3'], lanes=4, device='cpu', seed=1, packed=True)
  with pytest.raises(ValueError, match='keyed like envs'):
    batch.run_episodes({'catch': tr.stream_agent(batch.envs['catch'], 0)})
  with pytest.raises(ValueError, match='CUDA'):
    batch.run_host_episodes({k: None for k in batch.envs})
  steps = {k: env.steps_done for k, env in batch.envs.items()}
  assert batch.run_episodes(stream_agents(batch, 0), num_episodes=0) == {k: 0 for k in batch.envs}
  assert {k: env.steps_done for k, env in batch.envs.items()} == {k: n + 1 for k, n in steps.items()}
  batch.close()


# ----- refusals ---------------------------------------------------------------------------------------------------
def test_python_arguments_are_checked():
  env = bsuite_b200.load_from_id('catch/0', batch=4, device='cpu', seed=0)
  out, previous = env.make_buffers(), env.make_buffers()
  mask, left, actions = torch.ones(4, dtype=torch.bool), torch.ones(4, dtype=torch.int64), torch.zeros(4, dtype=torch.int32)
  with pytest.raises(ValueError, match='go together'):
    env.step(actions, out=out, mask=mask, episodes_left=left)
  with pytest.raises(ValueError, match='go together'):
    env.step(actions, out=out, mask=mask, previous=previous)
  with pytest.raises(ValueError, match='needs mask'):
    env.step(actions, out=out, episodes_left=left, previous=previous)
  with pytest.raises(ValueError, match='out='):
    env.step(actions, mask=mask, episodes_left=left, previous=previous)
  with pytest.raises(ValueError, match='contiguous'):
    env.step(actions, out=out, mask=torch.ones(8, dtype=torch.bool)[::2], episodes_left=left, previous=previous)
  with pytest.raises(ValueError, match='int64'):
    env.step(actions, out=out, mask=mask, episodes_left=left.int(), previous=previous)
  with pytest.raises(ValueError, match='StepBuffers'):
    env.step(actions, out=out, mask=mask, episodes_left=left, previous=previous.timestep())
  with pytest.raises(_lib.EngineError, match='own observation buffer'):
    env.step(actions, out=out, mask=mask, episodes_left=left, previous=out)
  same = bsuite_b200.load_from_id('catch/0', batch=4, device='cpu', seed=0, autoreset='same_step')
  with pytest.raises(_lib.EngineError, match='both output sets'):
    same.step(actions, out=same.make_buffers(final_observation=True), mask=mask, episodes_left=left,
              previous=same.make_buffers())
  with_final = same.make_buffers(final_observation=True)
  bad = bsuite_b200.environment.StepBuffers(out.observation, out.reward, out.discount, out.step_type,
                                            final_observation=with_final.final_observation)
  with pytest.raises(_lib.EngineError, match='SAME_STEP'):
    env.step(actions, out=bad, mask=mask, episodes_left=left,
             previous=bsuite_b200.environment.StepBuffers(previous.observation, previous.reward, previous.discount,
                                                          previous.step_type,
                                                          final_observation=torch.zeros_like(with_final.final_observation)))
  assert env.steps_done == 0 and same.steps_done == 0
  env.reset(out=out)
  env.step(actions, out=out, mask=mask, episodes_left=left, previous=previous)
  assert env.steps_done == 2 and mask.all()         # a bool mask is updated in place: budgets left, nothing cleared


def test_abi_statuses():
  lib = _lib.load()
  assert lib.bsb_abi_version() == 15
  cfg = _lib.Config()
  cfg.family, cfg.rows, cfg.columns, cfg.reward_scale = _lib.CATCH, 10, 5, 1.0
  handle = ctypes.c_void_p()
  _lib.check(lib.bsb_create(ctypes.byref(cfg), 3, _lib.DEVICE_HOST, 5, 0, ctypes.byref(handle)))

  def outputs(final=False):
    arrays = dict(observation=np.zeros((3, 50), np.float32), reward=np.zeros(3, np.float32),
                  discount=np.zeros(3, np.float32), step_type=np.zeros(3, np.int32),
                  final_observation=np.zeros((3, 50), np.float32))
    o = _lib.Outputs()
    for name in ('observation', 'reward', 'discount', 'step_type'):
      setattr(o, name, arrays[name].ctypes.data)
    if final:
      o.final_observation = arrays['final_observation'].ctypes.data
    return o, arrays

  (out, keep_out), (prev, keep_prev) = outputs(), outputs()
  mask, left, actions = np.ones(3, np.uint8), np.array([0, 1, 2], np.int64), np.zeros(3, np.int32)
  step = lib.bsb_step_budgeted
  args = [handle, actions.ctypes.data, mask.ctypes.data, left.ctypes.data, ctypes.byref(out), ctypes.byref(prev), None]
  for k in range(6):                               # every required pointer
    bad = list(args)
    bad[k] = None
    assert step(*bad) == 1
  assert b'bsb_step_budgeted needs' in lib.bsb_last_error()
  no_obs = _lib.Outputs.from_buffer_copy(prev)
  no_obs.observation = None
  assert step(*args[:5], ctypes.byref(no_obs), None) == 1
  assert step(*args[:5], ctypes.byref(out), None) == 1
  assert b'own observation buffer' in lib.bsb_last_error()
  final, keep_final = outputs(final=True)
  assert step(*args[:4], ctypes.byref(final), ctypes.byref(prev), None) == 1
  assert b'both output sets' in lib.bsb_last_error()
  final2, keep_final2 = outputs(final=True)
  assert step(*args[:4], ctypes.byref(final), ctypes.byref(final2), None) == 1
  assert b'SAME_STEP' in lib.bsb_last_error()
  steps = ctypes.c_int64()
  _lib.check(lib.bsb_steps_done(handle, ctypes.byref(steps)))
  assert steps.value == 0
  _lib.check(step(*args))
  _lib.check(lib.bsb_steps_done(handle, ctypes.byref(steps)))
  assert steps.value == 1
  assert mask.tolist() == [0, 1, 1] and left.tolist() == [0, 1, 2]      # lane 0 had no budget: it sat out
  del keep_out, keep_prev, keep_final, keep_final2
  _lib.check(lib.bsb_destroy(handle))


# ----- the GPU cases cover the list -------------------------------------------------------------------------------
def test_gpu_cases_cover_every_masked_kernel_of_the_list():
  """Every variant of the list, times its bit sources, has a case in test_budgeted_step_gpu.py: with it the
  CALL_BUDGETED instantiation of masked_kernel."""
  from tests import test_budgeted_step_gpu as g
  from tests import test_advance_gpu as a
  assert set(g.CASES) == set(a.CASES)
