"""Masked calls (BatchedEnvironment.reset / step with `mask`, bsb_reset_masked / bsb_step_masked) on the host path.

Lane i of a handle driven by masked calls must be, bit for bit, lane 0 of a one-lane handle with the same seed and
lane_offset + i driven by only the calls in which mask[i] was set: the same timesteps, bsuite_info(), episode
statistics and log rows.  Inactive lanes' output entries are never written."""
import ctypes

import numpy as np
import pytest
import torch

import bsuite_b200
from bsuite_b200 import _lib
from bsuite_b200 import rollouts
from bsuite_b200 import suite
from tests import conftest as cf
from tests import test_golden_parity as golden

DENSITIES = (0.0, 0.03, 0.5, 1.0)
SENTINEL = 7           # fills every output entry before a call: an inactive lane's entries must still hold it
FIELDS = ('observation', 'reward', 'discount', 'step_type', 'final_observation')


def make_plan(batch, calls, num_actions, seed, densities=DENSITIES, reset_every=7):
  """[(kind, mask bool [B], actions int32 [B])]: masks of the given densities in turn, a masked reset every
  `reset_every` calls; inactive lanes get out-of-range actions, which must never be read."""
  rng = np.random.default_rng(seed)
  plan = []
  for c in range(calls):
    mask = rng.random(batch) < densities[c % len(densities)]
    actions = rng.integers(0, num_actions, batch).astype(np.int32)
    actions[~mask] = np.where(rng.random(int((~mask).sum())) < 0.5, -3, num_actions + 5)
    plan.append(('reset' if c % reset_every == reset_every - 1 else 'step', mask, actions))
  return plan


def fill(out):
  for name in FIELDS:
    tensor = getattr(out, name)
    if tensor is not None:
      tensor.fill_(SENTINEL)


def masked_call(env, kind, mask, actions, out):
  mask_t = torch.as_tensor(mask).to(env.device)
  if kind == 'reset':
    return env.reset(out=out, mask=mask_t)
  return env.step(torch.as_tensor(actions).to(env.device), out=out, mask=mask_t)


def lane_rows(name, tensor, env):
  """`tensor` with the lane axis first (a ragged pack's flat observation: one row per lane of every setting)."""
  if env.ragged and name == 'observation':
    return [row.reshape(-1) for part in env.split_observation(tensor.cpu()) for row in part]
  return tensor.cpu()


def drive(env, plan, final_observation=False):
  """Runs `plan` on `env` with masked calls; returns {field: [calls] of per-lane rows (None where inactive)}."""
  out = env.make_buffers(final_observation=final_observation)
  got = {name: [] for name in FIELDS}
  for kind, mask, actions in plan:
    fill(out)
    masked_call(env, kind, mask, actions, out)
    for name in FIELDS:
      tensor = getattr(out, name)
      if tensor is None:
        continue
      rows = lane_rows(name, tensor, env)
      for i in np.flatnonzero(~mask):
        assert torch.all(rows[i] == SENTINEL), f'{name} of inactive lane {i} was written'
      got[name].append([rows[i].clone() if mask[i] else None for i in range(len(mask))])
  return got


def plain_call(env, kind, action, out):
  if kind == 'reset':
    return env.reset(out=out)
  return env.step(torch.tensor([action], dtype=torch.int32).to(env.device), out=out)


def accumulators(env):
  acc = {f'info {k}': v.cpu() for k, v in env.bsuite_info().items()}
  if env._track:
    acc.update({f'stat {k}': v.cpu() for k, v in env.episode_stats().items()})
  if env._log_schedule is not None:
    rows = env.logged_rows()
    acc['log rows'] = rows['rows'].cpu()
    acc['log counts'] = rows['counts'].cpu()
  return acc


def lane_of(acc, i):
  return {k: v[..., i:i + 1] for k, v in acc.items()}


def check_against_one_lane(env, plan, got, one_lane, final_observation=False, lanes=None):
  """Lane i of `env` (driven by `plan`, results `got`) against `one_lane(i)` driven by lane i's own calls."""
  acc = accumulators(env)
  for i in (range(env.batch) if lanes is None else lanes):
    ref = one_lane(i)
    out = ref.make_buffers(final_observation=final_observation)
    c_own = 0
    for c, (kind, mask, actions) in enumerate(plan):
      if not mask[i]:
        continue
      fill(out)
      plain_call(ref, kind, int(actions[i]), out)
      c_own += 1
      for name in FIELDS:
        tensor = getattr(out, name)
        if tensor is not None:
          assert torch.equal(got[name][c][i], tensor[0].cpu()), f'{name} of lane {i} at call {c} differs'
    assert ref.steps_done == c_own
    want, have = accumulators(ref), lane_of(acc, i)
    for key in want:
      assert torch.equal(have[key], want[key]), f'{key} of lane {i} differs'
  assert env.steps_done == len(plan)


def _mnist_if_needed(bsuite_id, request):
  if bsuite_id.startswith('mnist'):
    request.getfixturevalue('mnist_dir')


@pytest.mark.parametrize('bsuite_id', suite.one_per_experiment())
def test_every_experiment_matches_one_lane_handles(bsuite_id, request):
  _mnist_if_needed(bsuite_id, request)
  B, seed = 9, 11
  env = bsuite_b200.load_from_id(bsuite_id, batch=B, device='cpu', seed=seed, lane_offset=3, track_episodes=True,
                                 record_rows=True)
  plan = make_plan(B, 48, env.num_actions, seed=sum(map(ord, bsuite_id)))
  got = drive(env, plan)
  check_against_one_lane(env, plan, got, lambda i: bsuite_b200.load_from_id(
      bsuite_id, batch=1, device='cpu', seed=seed, lane_offset=3 + i, track_episodes=True, record_rows=True))


@pytest.mark.parametrize('bsuite_id,kwargs', [
    ('catch/0', dict(autoreset='same_step')),
    ('deep_sea/2', dict(autoreset='same_step', obs_dtype='bfloat16')),
    ('umbrella_distract/3', dict(autoreset='same_step')),
    ('cartpole_swingup/4', dict(autoreset='same_step', obs_dtype='bfloat16')),
    ('mnist/0', dict(autoreset='same_step', obs_dtype='bfloat16')),
    ('memory_len/2', dict(autoreset='same_step')),
    ('deep_sea/0', dict(obs_dtype='uint8')),
    ('catch/0', dict(obs_dtype='uint8')),
    ('mountain_car/0', dict(obs_dtype='bfloat16')),
    ('catch/0', dict(rng='mt19937')),
    ('deep_sea_stochastic/1', dict(rng='mt19937')),
    ('umbrella_distract/2', dict(rng='mt19937')),
    ('cartpole_noise/3', dict(rng='mt19937')),
    ('mountain_car_noise/2', {}),
    ('bandit_noise/1', dict(reward_dtype='float64')),
])
def test_handle_kinds_match_one_lane_handles(bsuite_id, kwargs, request):
  _mnist_if_needed(bsuite_id, request)
  B, seed = 7, 5
  same_step = kwargs.get('autoreset') == 'same_step'
  kw = dict(track_episodes=True, record_rows=not kwargs.get('rng'), **kwargs)
  env = bsuite_b200.load_from_id(bsuite_id, batch=B, device='cpu', seed=seed, **kw)
  plan = make_plan(B, 60, env.num_actions, seed=len(bsuite_id), densities=(0.5, 1.0, 0.03, 0.7), reset_every=13)
  got = drive(env, plan, final_observation=same_step)
  check_against_one_lane(env, plan, got, lambda i: bsuite_b200.load_from_id(
      bsuite_id, batch=1, device='cpu', seed=seed, lane_offset=i, **kw), final_observation=same_step)


def packed_parts(name, lanes, ragged, seed=4):
  pack = bsuite_b200.load_experiment(name, lanes, device='cpu', seed=seed, track_episodes=True, record_rows=True,
                                     ragged=ragged)
  parts = [bsuite_b200.load_from_id(bsuite_id, batch=lanes, device='cpu', seed=s, track_episodes=True,
                                    record_rows=True) for bsuite_id, s in zip(pack.bsuite_ids, pack.setting_seeds)]
  return pack, parts


@pytest.mark.parametrize('name,ragged', [('catch', False), ('cartpole_noise', False), ('bandit', False),
                                         ('memory_len', False), ('umbrella_length', False), ('mnist_scale', False),
                                         ('deep_sea', True), ('memory_size', True), ('umbrella_distract', True)])
def test_packed_and_ragged_match_separate_handles(name, ragged, request):
  if name.startswith('mnist'):
    request.getfixturevalue('mnist_dir')
  lanes = 3
  pack, parts = packed_parts(name, lanes, ragged)
  plan = make_plan(pack.batch, 40, pack.num_actions, seed=len(name))
  got = drive(pack, plan)
  acc = accumulators(pack)
  for k, part in enumerate(parts):
    sl = slice(k * lanes, (k + 1) * lanes)
    sub = [(kind, mask[sl], actions[sl]) for kind, mask, actions in plan]
    part_got = drive(part, sub)
    for name_ in FIELDS:
      for c in range(len(plan)):
        for j in range(lanes):
          a, b = got[name_][c][sl.start + j] if got[name_] else None, part_got[name_][c][j] if part_got[name_] else None
          assert (a is None and b is None) or torch.equal(a.reshape(-1), b.reshape(-1)), f'{name_} of setting {k} lane {j} at call {c}'
    for key, value in accumulators(part).items():
      assert torch.equal(acc[key][..., sl], value), f'{key} of setting {k}'


def test_full_mask_equals_plain_calls():
  for bsuite_id in ('catch/0', 'cartpole/0', 'deep_sea/1'):
    a = bsuite_b200.load_from_id(bsuite_id, batch=6, device='cpu', seed=1, track_episodes=True, record_rows=True)
    b = bsuite_b200.load_from_id(bsuite_id, batch=6, device='cpu', seed=1, track_episodes=True, record_rows=True)
    out_a, out_b = a.make_buffers(), b.make_buffers()
    ones = torch.ones(6, dtype=torch.bool)
    rng = np.random.default_rng(0)
    for c in range(40):
      actions = torch.as_tensor(rng.integers(0, a.num_actions, 6).astype(np.int32))
      if c % 11 == 5:
        a.reset(out=out_a, mask=ones)
        b.reset(out=out_b)
      else:
        a.step(actions, out=out_a, mask=ones.to(torch.uint8))
        b.step(actions, out=out_b)
      for name in ('observation', 'reward', 'discount', 'step_type'):
        assert torch.equal(getattr(out_a, name), getattr(out_b, name))
    for key, value in accumulators(b).items():
      assert torch.equal(accumulators(a)[key], value), key
    assert a.state_dict()['blob'].tobytes() == b.state_dict()['blob'].tobytes()


def test_sitting_out_before_the_first_call_keeps_logging_columns_exact():
  """A lane that sits out calls before its first one reads steps = episode_len = 0 until it makes its own call."""
  env = bsuite_b200.load_from_id('catch/0', batch=2, device='cpu', seed=0, track_episodes=True)
  out = env.make_buffers()
  only0 = torch.tensor([True, False])
  env.reset(out=out, mask=only0)
  for _ in range(4):
    env.step(torch.zeros(2, dtype=torch.int32), out=out, mask=only0)
  stats = env.episode_stats()
  assert stats['steps'][1] == 0 and stats['episode_len'][1] == 0 and stats['episode'][1] == 0
  assert stats['steps'][0] == 4 and stats['episode_len'][0] == 4
  env.step(torch.zeros(2, dtype=torch.int32), out=out, mask=torch.tensor([False, True]))
  stats = env.episode_stats()
  assert stats['steps'][1] == 0 and stats['episode_len'][1] == 0 and out.step_type[1] == 0
  assert stats['steps'][0] == 4 and stats['episode_len'][0] == 4


def test_state_dict_round_trip_in_a_masked_sequence():
  env = bsuite_b200.load_from_id('cartpole_noise/2', batch=5, device='cpu', seed=2, track_episodes=True,
                                 record_rows=True)
  plan = make_plan(5, 50, env.num_actions, seed=9)
  drive(env, plan[:20])
  state = env.state_dict()
  first = drive(env, plan[20:])
  acc_first = accumulators(env)
  env.load_state_dict(state)
  assert env.steps_done == 20
  again = drive(env, plan[20:])
  for name in FIELDS:
    for c in range(len(first[name])):
      for a, b in zip(first[name][c], again[name][c]):
        assert (a is None and b is None) or torch.equal(a, b)
  for key, value in accumulators(env).items():
    assert torch.equal(acc_first[key], value), key


@pytest.mark.parametrize('name', cf.golden_case_names())
def test_golden_fixtures_with_lanes_at_their_own_pace(name, mnist_dir):
  """Every fixture lane advances only where a random mask selects it, its `reset_at` resets issued as masked
  resets; each lane must still reproduce its recorded trace."""
  del mnist_dir
  meta, data = cf.load_golden(name)
  kwargs = dict(meta['kwargs'])
  if meta['wrapper'] == 'noise':
    kwargs['noise_scale'] = meta['wrapper_arg']
  elif meta['wrapper'] == 'scale':
    kwargs['reward_scale'] = meta['wrapper_arg']
  B = len(meta['lanes'])
  env = bsuite_b200.make(meta['env_class'], batch=B, device='cpu', seed=meta['seed'], rng=meta['rng'],
                         engine_kwargs=dict(reward_dtype='float64'), **kwargs)
  actions = data['actions']
  T = actions.shape[0]
  reset_at = set(meta['reset_at'])
  pos = np.zeros(B, dtype=np.int64)         # each lane's next call in the fixture
  res = {k: np.zeros(data[k].shape, dtype=np.float64 if k != 'step_type' else np.int32)
         for k in ('step_type', 'reward', 'discount')}
  res['observation'] = np.zeros(data['observation'].shape, dtype=np.float32)
  out = env.make_buffers()
  rng = np.random.default_rng(len(name))
  while (pos < T).any():
    kind = 'reset' if rng.random() < 0.5 else 'step'
    due = (pos < T) & np.array([(p in reset_at) == (kind == 'reset') for p in pos])
    mask = due & (rng.random(B) < 0.6)
    acts = np.array([actions[min(p, T - 1), i] for i, p in enumerate(pos)], dtype=np.int32)
    masked_call(env, kind, mask, acts, out)
    for i in np.flatnonzero(mask):
      for k in ('step_type', 'reward', 'discount'):
        res[k][pos[i], i] = getattr(out, k)[i].item()
      res['observation'][pos[i], i] = out.observation[i].numpy().reshape(res['observation'][pos[i], i].shape)
    pos += mask
  res['observation'] = res['observation'].reshape((T, B) + tuple(env.obs_shape))
  res['info'] = {k: v.numpy() for k, v in env.bsuite_info().items()}
  res['host'] = True
  golden._compare(meta, data, res)


def _first_lane_loop(bsuite_id, lane, num_episodes, policy):
  env = bsuite_b200.load_from_id(bsuite_id, batch=1, device='cpu', seed=3, lane_offset=lane, record_rows=True)
  for _ in range(num_episodes):
    ts = env.reset()
    while int(ts.step_type[0]) != 2:
      ts = env.step(policy(ts.observation))
  return env


class ObservationPolicy:
  """A deterministic policy of each lane's own observation."""

  def __init__(self, num_actions):
    self.num_actions = num_actions

  def __call__(self, observation):
    flat = observation.reshape(observation.shape[0], -1).to(torch.float64)
    weights = torch.arange(1, flat.shape[1] + 1, dtype=torch.float64)
    return ((flat * weights).sum(1) * 1000).floor().to(torch.int64).remainder(self.num_actions).to(torch.int32)

  def select_action(self, timestep):
    return self(timestep.observation)

  def update(self, timestep, action, new_timestep):
    del timestep, action, new_timestep


@pytest.mark.parametrize('bsuite_id', ['cartpole/0', 'catch/0', 'mountain_car_scale/1'])
def test_run_episodes_plays_each_lanes_budget(bsuite_id):
  B, episodes = 4, 3
  env = bsuite_b200.load_from_id(bsuite_id, batch=B, device='cpu', seed=3, record_rows=True)
  policy = ObservationPolicy(env.num_actions)
  rollouts.run_episodes(policy, env, num_episodes=episodes, check_every=5)
  acc = accumulators(env)
  assert torch.all(acc['stat episode'] == episodes)
  for i in range(B):
    ref = _first_lane_loop(bsuite_id, i, episodes, policy)
    for key, value in accumulators(ref).items():
      assert torch.equal(lane_of(acc, i)[key], value), f'{key} of lane {i}'


def test_run_episodes_uses_each_settings_budget_on_packed_handles():
  pack = bsuite_b200.load_experiment('cartpole', 2, settings=[0, 1], device='cpu', seed=1, track_episodes=True)
  budgets = [spec.bsuite_num_episodes for spec in pack._pack[1]]
  small = [2, 3]
  for spec, n in zip(pack._pack[1], small):     # a short run: each setting's budget lowered in place
    spec.bsuite_num_episodes = n
  try:
    rollouts.run_episodes(ObservationPolicy(pack.num_actions), pack)
  finally:
    for spec, n in zip(pack._pack[1], budgets):
      spec.bsuite_num_episodes = n
  assert pack.episode_stats()['episode'].tolist() == [2.0, 2.0, 3.0, 3.0]


def test_mask_arguments_are_checked():
  env = bsuite_b200.load_from_id('catch/0', batch=4, device='cpu', seed=0)
  out = env.make_buffers()
  actions = torch.zeros(4, dtype=torch.int32)
  with pytest.raises(ValueError, match='out='):
    env.step(actions, mask=torch.ones(4, dtype=torch.bool))
  with pytest.raises(ValueError, match='out='):
    env.reset(mask=torch.ones(4, dtype=torch.bool))
  with pytest.raises(ValueError, match='shape'):
    env.step(actions, out=out, mask=torch.ones(5, dtype=torch.bool))
  with pytest.raises(ValueError, match='bool or uint8'):
    env.step(actions, out=out, mask=torch.ones(4, dtype=torch.int32))
  with pytest.raises(ValueError, match='bool or uint8'):
    env.reset(out=out, mask=[1, 1, 1, 1])
  env.reset(out=out, mask=torch.ones(4, dtype=torch.bool))
  with pytest.raises(_lib.EngineError, match='active lane 2'):      # an active lane's action is validated
    env.step(torch.tensor([0, 1, 9, 0], dtype=torch.int32), out=out, mask=torch.tensor([1, 1, 1, 0], dtype=torch.uint8))
  env.step(torch.tensor([0, 1, 2, 9], dtype=torch.int32), out=out, mask=torch.tensor([1, 1, 1, 0], dtype=torch.uint8))


def test_abi_statuses():
  lib = _lib.load()
  cfg = _lib.Config()
  cfg.family, cfg.rows, cfg.columns, cfg.reward_scale = _lib.CATCH, 10, 5, 1.0
  handle = ctypes.c_void_p()
  _lib.check(lib.bsb_create(ctypes.byref(cfg), 3, _lib.DEVICE_HOST, 5, 0, ctypes.byref(handle)))
  obs = np.zeros((3, 50), np.float32)
  final = np.zeros((3, 50), np.float32)
  out = _lib.Outputs()
  out.observation = obs.ctypes.data
  mask = np.array([1, 0, 1], np.uint8)
  actions = np.array([0, 7, 1], np.int32)
  assert lib.bsb_reset_masked(handle, None, ctypes.byref(out), None) == 1
  assert lib.bsb_reset_masked(None, mask.ctypes.data, ctypes.byref(out), None) == 1
  assert lib.bsb_step_masked(handle, None, mask.ctypes.data, ctypes.byref(out), None) == 1
  assert lib.bsb_step_masked(handle, actions.ctypes.data, None, ctypes.byref(out), None) == 1
  empty = _lib.Outputs()
  assert lib.bsb_step_masked(handle, actions.ctypes.data, mask.ctypes.data, ctypes.byref(empty), None) == 1
  out.final_observation = final.ctypes.data      # next-step handle
  assert lib.bsb_step_masked(handle, actions.ctypes.data, mask.ctypes.data, ctypes.byref(out), None) == 1
  assert b'SAME_STEP' in lib.bsb_last_error()
  out.final_observation = None
  _lib.check(lib.bsb_reset_masked(handle, mask.ctypes.data, ctypes.byref(out), None))
  _lib.check(lib.bsb_step_masked(handle, actions.ctypes.data, mask.ctypes.data, ctypes.byref(out), None))
  actions[0] = -1
  assert lib.bsb_step_masked(handle, actions.ctypes.data, mask.ctypes.data, ctypes.byref(out), None) == 1
  steps = ctypes.c_int64()
  _lib.check(lib.bsb_steps_done(handle, ctypes.byref(steps)))
  assert steps.value == 2
  assert not obs[1].any()                         # lane 1 never made a call
  _lib.check(lib.bsb_destroy(handle))
