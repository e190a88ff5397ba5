"""Masked rollouts (BatchedEnvironment.rollout with `mask` / `episodes_left`, bsb_rollout_masked) on the host path.

One masked rollout of T steps must equal, bit for bit, T masked steps on a twin handle in which lane i is active at
step t while its mask is set and its budget is positive, each LAST taking one from the budget: every output entry
written (unwritten ones keep a sentinel), the actions used, steps_done, the budgets, bsuite_info(), episode
statistics, log rows and the raw state.  `run_random_episodes` must equal `run_episodes` driven by the host mirror
of the on-device action sampler."""
import ctypes

import numpy as np
import pytest
import torch

import bsuite_b200
from bsuite_b200 import _lib
from bsuite_b200 import analysis
from bsuite_b200 import rollouts
from bsuite_b200 import suite
from tests import gauss_draw_reference as gauss
from tests import test_masked as tm

SENTINEL = tm.SENTINEL
FIELDS = tm.FIELDS + ('actions',)
LAST = 2


def make_launches(batch, num_actions, seed, densities=(1.0, 0.0, 0.5, 0.03, 1.0, 0.5), steps=(5, 3, 9, 1, 16, 7)):
  """[(T, mask bool [B], budgets int64 [B] or None, actions int32 [T, B] or None)]: the densities in turn, budgets
  of 0 to 3 episodes (every other launch none), explicit actions every other launch (out-of-range where the mask is
  clear: they must never be read), else sampled ones."""
  rng = np.random.default_rng(seed)
  launches = []
  for k, (density, T) in enumerate(zip(densities, steps)):
    mask = rng.random(batch) < density
    budgets = rng.integers(0, 4, batch).astype(np.int64) if k % 2 == 0 else None
    actions = None
    if k % 3 != 1:
      actions = rng.integers(0, num_actions, (T, batch)).astype(np.int32)
      actions[:, ~mask] = np.where(rng.random((T, int((~mask).sum()))) < 0.5, -3, num_actions + 5)
    launches.append((T, mask, budgets, actions))
  return launches


def fill(out):
  for name in FIELDS:
    tensor = getattr(out, name, None)
    if tensor is not None:
      tensor.fill_(SENTINEL)


def rollout_launch(env, launch, out, action_seed):
  """One masked rollout of `launch`; returns the budgets after it (or None)."""
  T, mask, budgets, actions = launch
  left = None if budgets is None else torch.tensor(budgets).to(env.device)      # a copy: the launch updates it
  fill(out)
  env.rollout(T, actions=None if actions is None else torch.as_tensor(actions).to(env.device), action_seed=action_seed,
              out=out, mask=torch.as_tensor(mask).to(env.device), episodes_left=left)
  return None if left is None else left.cpu().numpy()


def stepped_launch(env, launch, action_seed, final_observation):
  """The same launch as masked steps: ({field: [T] tensors}, budgets after it)."""
  T, mask, budgets, actions = launch
  left = None if budgets is None else budgets.copy()
  out = env.make_buffers(final_observation=final_observation)
  got = {name: [] for name in FIELDS}
  for t in range(T):
    active = mask & (left > 0) if left is not None else mask.copy()
    if actions is not None:
      step_actions = actions[t]
    else:
      step_actions = env.random_actions(1, action_seed, first_step=env.steps_done)[0]
    fill(out)
    env.step(torch.as_tensor(step_actions).to(env.device), out=out, mask=torch.as_tensor(active).to(env.device))
    for name in tm.FIELDS:
      tensor = getattr(out, name)
      if tensor is not None:
        got[name].append(tensor.cpu().clone())
    acts = torch.full((env.batch,), SENTINEL, dtype=torch.int32)
    acts[torch.as_tensor(active)] = torch.as_tensor(np.asarray(step_actions, dtype=np.int32))[torch.as_tensor(active)]
    got['actions'].append(acts)
    if left is not None:
      left -= (active & (out.step_type.cpu().numpy() == LAST)).astype(np.int64)
  return got, left


def raw_state(env):
  """The state_dict() blob with every gaussian cache whose flag is clear zeroed: a fused launch stores a lane's
  streams once, so a value cached and consumed within it never reaches memory, where T single calls leave it
  behind unread."""
  blob = env.state_dict()['blob'].copy()
  try:
    sections = gauss.blob_sections(env)
  except (AssertionError, KeyError, AttributeError):
    return blob.tobytes()
  for pos, cache in (('rng_pos', 'rng_gauss'), ('wrng_pos', 'wrng_gauss')):
    if cache in sections:
      stale = (gauss.section(blob, sections, pos) & np.uint64(gauss.HASGAUSS)) == 0
      gauss.put_section(blob, sections, cache, np.where(stale, 0.0, gauss.section(blob, sections, cache)))
  return blob.tobytes()


def check_launches(env, twin, launches, action_seed=5, final_observation=False):
  """Runs every launch on `env` as one masked rollout and on `twin` as masked steps, and compares after each."""
  for launch in launches:
    T = launch[0]
    out = env.make_buffers(T, with_actions=True, final_observation=final_observation)
    left = rollout_launch(env, launch, out, action_seed)
    want, want_left = stepped_launch(twin, launch, action_seed, final_observation)
    for name in FIELDS:
      tensor = getattr(out, name)
      if tensor is None:
        continue
      for t in range(T):
        assert torch.equal(tensor[t].cpu(), want[name][t]), f'{name} at step {t} of a {T}-step launch differs'
    if left is not None:
      assert np.array_equal(left, want_left)
    assert env.steps_done == twin.steps_done
    acc, acc_twin = tm.accumulators(env), tm.accumulators(twin)
    for key in acc_twin:
      assert torch.equal(acc[key], acc_twin[key]), key
    assert raw_state(env) == raw_state(twin)


def twins(bsuite_id, batch, seed=7, **kwargs):
  kw = dict(batch=batch, device='cpu', seed=seed, track_episodes=True, **kwargs)
  return bsuite_b200.load_from_id(bsuite_id, **kw), bsuite_b200.load_from_id(bsuite_id, **kw)


@pytest.mark.parametrize('bsuite_id', suite.one_per_experiment())
def test_every_experiment_equals_masked_steps(bsuite_id, request):
  tm._mnist_if_needed(bsuite_id, request)
  env, twin = twins(bsuite_id, 37, lane_offset=3, record_rows=True)
  launches = make_launches(env.batch, env.num_actions, seed=sum(map(ord, bsuite_id)))
  check_launches(env, twin, launches)


@pytest.mark.parametrize('bsuite_id,kwargs', [
    ('catch/0', dict(autoreset='same_step')),
    ('deep_sea/2', dict(autoreset='same_step', obs_dtype='bfloat16')),
    ('umbrella_distract/3', dict(autoreset='same_step')),
    ('bandit/0', dict(autoreset='same_step')),
    ('mnist/0', dict(autoreset='same_step', obs_dtype='bfloat16')),
    ('catch/0', dict(autoreset='same_step', obs_dtype='uint8')),
    ('deep_sea/0', dict(obs_dtype='uint8')),
    ('mountain_car/0', dict(obs_dtype='bfloat16')),
    ('catch/0', dict(rng='mt19937')),
    ('deep_sea_stochastic/1', dict(rng='mt19937')),
    ('cartpole_noise/3', dict(rng='mt19937')),
    ('mountain_car_noise/2', {}),
    ('bandit_noise/1', dict(reward_dtype='float64')),
    ('catch_scale/2', {}),
])
def test_handle_kinds_equal_masked_steps(bsuite_id, kwargs, request):
  tm._mnist_if_needed(bsuite_id, request)
  same_step = kwargs.get('autoreset') == 'same_step'
  env, twin = twins(bsuite_id, 35, record_rows=not kwargs.get('rng'), **kwargs)
  launches = make_launches(env.batch, env.num_actions, seed=len(bsuite_id) + 1)
  check_launches(env, twin, launches, final_observation=same_step)


@pytest.mark.parametrize('name,ragged', [('catch', False), ('cartpole_noise', False), ('bandit', False),
                                         ('memory_len', False), ('umbrella_length', False), ('mnist_scale', False),
                                         ('deep_sea', True), ('memory_size', True), ('umbrella_distract', True)])
def test_packed_and_ragged_equal_masked_steps(name, ragged, request):
  if name.startswith('mnist'):
    request.getfixturevalue('mnist_dir')
  kw = dict(device='cpu', seed=4, track_episodes=True, record_rows=True, ragged=ragged)
  env, twin = bsuite_b200.load_experiment(name, 5, **kw), bsuite_b200.load_experiment(name, 5, **kw)
  check_launches(env, twin, make_launches(env.batch, env.num_actions, seed=len(name)))


def test_two_shards_equal_one_handle():
  B, half = 40, 20
  kw = dict(device='cpu', seed=9, track_episodes=True, record_rows=True)
  whole = bsuite_b200.load_from_id('catch/1', batch=B, **kw)
  shards = [bsuite_b200.load_from_id('catch/1', batch=half, lane_offset=k * half, **kw) for k in range(2)]
  for T, mask, budgets, actions in make_launches(B, whole.num_actions, seed=3):
    out = whole.make_buffers(T, with_actions=True)
    left = rollout_launch(whole, (T, mask, budgets, actions), out, action_seed=11)
    for k, shard in enumerate(shards):
      sl = slice(k * half, (k + 1) * half)
      part = (T, mask[sl], None if budgets is None else budgets[sl], None if actions is None else actions[:, sl])
      shard_out = shard.make_buffers(T, with_actions=True)
      shard_left = rollout_launch(shard, part, shard_out, action_seed=11)
      for name in FIELDS:
        if getattr(out, name) is not None:
          assert torch.equal(getattr(out, name)[:, sl], getattr(shard_out, name)), name
      if left is not None:
        assert np.array_equal(left[sl], shard_left)
  acc = tm.accumulators(whole)
  for k, shard in enumerate(shards):
    for key, value in tm.accumulators(shard).items():
      assert torch.equal(acc[key][..., k * half:(k + 1) * half], value), key


def test_state_dict_round_trip_between_launches():
  env = bsuite_b200.load_from_id('cartpole_noise/2', batch=33, device='cpu', seed=2, track_episodes=True,
                                 record_rows=True)
  launches = make_launches(33, env.num_actions, seed=8)
  for launch in launches[:2]:
    rollout_launch(env, launch, env.make_buffers(launch[0], with_actions=True), action_seed=1)
  state = env.state_dict()

  def rest():
    outs, lefts = [], []
    for launch in launches[2:]:
      out = env.make_buffers(launch[0], with_actions=True)
      lefts.append(rollout_launch(env, launch, out, action_seed=1))
      outs.append(out)
    return outs, lefts, tm.accumulators(env), raw_state(env)

  first = rest()
  env.load_state_dict(state)
  again = rest()
  for a, b in zip(first[0], again[0]):
    for name in FIELDS:
      if getattr(a, name) is not None:
        assert torch.equal(getattr(a, name), getattr(b, name)), name
  for a, b in zip(first[1], again[1]):
    assert (a is None and b is None) or np.array_equal(a, b)
  for key in first[2]:
    assert torch.equal(first[2][key], again[2][key]), key
  assert first[3] == again[3]


def test_budgets_stop_lanes_mid_launch():
  """Same-step bandit lanes finish an episode at every step: a budget of k stops its lane after exactly k steps of a
  longer launch."""
  env = bsuite_b200.load_from_id('bandit/0', batch=6, device='cpu', seed=0, track_episodes=True, autoreset='same_step')
  env.reset(out=env.make_buffers(), mask=torch.ones(6, dtype=torch.bool))
  left = torch.tensor([0, 1, 2, 3, 5, 9], dtype=torch.int64)
  out = env.make_buffers(6, with_actions=True)
  fill(out)
  env.rollout(6, out=out, mask=torch.tensor([1, 1, 1, 1, 1, 0], dtype=torch.uint8), episodes_left=left)
  assert left.tolist() == [0, 0, 0, 0, 0, 9]
  written = (out.step_type != SENTINEL).sum(0).tolist()
  assert written == [0, 1, 2, 3, 5, 0]
  assert env.episode_stats()['episode'].tolist() == [0, 1, 2, 3, 5, 0]
  assert env.steps_done == 7


def stream_agent(env, action_seed):
  class StreamAgent:
    def select_action(self, timestep):
      del timestep
      return torch.as_tensor(env.random_actions(1, action_seed, first_step=env.steps_done)[0]).to(env.device)

    def update(self, timestep, action, new_timestep):
      del timestep, action, new_timestep
  return StreamAgent()


def check_random_episodes(env, twin, num_episodes=None, action_seed=3):
  calls = rollouts.run_random_episodes(env, num_episodes, action_seed=action_seed, steps_per_launch=8)
  assert calls % 8 == 0
  rollouts.run_episodes(stream_agent(twin, action_seed), twin, num_episodes, check_every=5)
  acc, acc_twin = tm.accumulators(env), tm.accumulators(twin)
  for key in acc_twin:
    assert torch.equal(acc[key], acc_twin[key]), key


@pytest.mark.parametrize('bsuite_id', suite.one_per_experiment())
def test_run_random_episodes_equals_run_episodes(bsuite_id, request):
  tm._mnist_if_needed(bsuite_id, request)
  env, twin = twins(bsuite_id, 5, lane_offset=2, record_rows=True)
  check_random_episodes(env, twin, num_episodes=2)
  assert torch.all(env.episode_stats()['episode'] == 2)


def test_run_random_episodes_uses_each_settings_budget_and_scores_equal():
  kw = dict(device='cpu', seed=1, track_episodes=True, record_rows=True)
  env, twin = bsuite_b200.load_experiment('bandit', 3, **kw), bsuite_b200.load_experiment('bandit', 3, **kw)
  specs = list(env._pack[1]) + [spec for spec in twin._pack[1] if all(spec is not s for s in env._pack[1])]
  budgets = [spec.bsuite_num_episodes for spec in specs]
  small = [3 + k % 4 for k in range(len(env._pack[1]))]
  for k, spec in enumerate(specs):             # a short run: each setting's budget lowered in place
    spec.bsuite_num_episodes = small[k % len(small)]
  try:
    check_random_episodes(env, twin)
  finally:
    for spec, n in zip(specs, budgets):
      spec.bsuite_num_episodes = n
  assert env.episode_stats()['episode'].tolist() == [float(n) for n in small for _ in range(3)]
  a, b = analysis.bsuite_score(env), analysis.bsuite_score(twin)
  assert torch.equal(a.score.view(torch.int64), b.score.view(torch.int64))      # bit for bit, NaN for absent ones
  assert torch.equal(a.finished, b.finished)
  assert torch.equal(a.tag_score.view(torch.int64), b.tag_score.view(torch.int64))
  assert not torch.isnan(a.score[0]).any()


def test_run_episodes_is_unchanged_by_the_shared_budget():
  env = bsuite_b200.load_from_id('catch/0', batch=3, device='cpu', seed=0, track_episodes=True)
  assert rollouts.episode_budget(env).tolist() == [env.bsuite_num_episodes] * 3
  assert rollouts.episode_budget(env, 4).tolist() == [4] * 3
  with pytest.raises(ValueError, match='steps_per_launch'):
    rollouts.run_random_episodes(env, 1, steps_per_launch=0)


def test_rollout_mask_arguments_are_checked():
  env = bsuite_b200.load_from_id('catch/0', batch=4, device='cpu', seed=0)
  out = env.make_buffers(3)
  ones = torch.ones(4, dtype=torch.bool)
  left = torch.ones(4, dtype=torch.int64)
  with pytest.raises(ValueError, match='out='):
    env.rollout(3, mask=ones)
  with pytest.raises(ValueError, match='episodes_left needs mask='):
    env.rollout(3, out=out, episodes_left=left)
  with pytest.raises(ValueError, match='shape'):
    env.rollout(3, out=out, mask=torch.ones(5, dtype=torch.bool))
  with pytest.raises(ValueError, match='bool or uint8'):
    env.rollout(3, out=out, mask=torch.ones(4, dtype=torch.int32))
  with pytest.raises(ValueError, match='int64'):
    env.rollout(3, out=out, mask=ones, episodes_left=torch.ones(4, dtype=torch.int32))
  with pytest.raises(ValueError, match='int64'):
    env.rollout(3, out=out, mask=ones, episodes_left=[1, 1, 1, 1])
  with pytest.raises(ValueError, match='shape'):
    env.rollout(3, out=out, mask=ones, episodes_left=torch.ones(5, dtype=torch.int64))
  with pytest.raises(ValueError, match='contiguous'):
    env.rollout(3, out=out, mask=ones, episodes_left=torch.ones(8, dtype=torch.int64)[::2])
  # an active lane's action is validated at every step, even after its budget would have stopped it
  left = torch.tensor([1, 1, 1, 1], dtype=torch.int64)
  bad = torch.zeros((3, 4), dtype=torch.int32)
  bad[2, 1] = 9
  state = raw_state(env)
  with pytest.raises(_lib.EngineError, match='active lane 1 at step 2'):
    env.rollout(3, actions=bad, out=out, mask=ones, episodes_left=left)
  assert raw_state(env) == state and left.tolist() == [1, 1, 1, 1] and env.steps_done == 0
  env.rollout(3, actions=bad, out=out, mask=torch.tensor([1, 0, 1, 1], dtype=torch.uint8), episodes_left=left)
  assert env.steps_done == 3


def test_abi_statuses():
  lib = _lib.load()
  assert lib.bsb_abi_version() == 15
  cfg = _lib.Config()
  cfg.family, cfg.rows, cfg.columns, cfg.reward_scale = _lib.CATCH, 10, 5, 1.0
  handle = ctypes.c_void_p()
  _lib.check(lib.bsb_create(ctypes.byref(cfg), 3, _lib.DEVICE_HOST, 5, 0, ctypes.byref(handle)))
  T = 4
  obs = np.zeros((T, 3, 50), np.float32)
  final = np.zeros((T, 3, 50), np.float32)
  out = _lib.Outputs()
  out.observation = obs.ctypes.data
  mask = np.array([1, 0, 1], np.uint8)
  left = np.array([2, 2, 0], np.int64)
  actions = np.zeros((T, 3), np.int32)
  actions[:, 1] = 7                             # lane 1 is masked out: never read
  rollout = lib.bsb_rollout_masked
  assert rollout(handle, T, actions.ctypes.data, 0, None, left.ctypes.data, ctypes.byref(out), None, None) == 1
  assert rollout(None, T, actions.ctypes.data, 0, mask.ctypes.data, None, ctypes.byref(out), None, None) == 1
  assert rollout(handle, T, None, 0, mask.ctypes.data, None, None, None, None) == 1
  empty = _lib.Outputs()
  assert rollout(handle, T, None, 0, mask.ctypes.data, None, ctypes.byref(empty), None, None) == 1
  assert rollout(handle, 0, None, 0, mask.ctypes.data, None, ctypes.byref(out), None, None) == 1
  assert rollout(handle, -2, None, 0, mask.ctypes.data, None, ctypes.byref(out), None, None) == 1
  out.final_observation = final.ctypes.data      # next-step handle
  assert rollout(handle, T, None, 0, mask.ctypes.data, None, ctypes.byref(out), None, None) == 1
  assert b'SAME_STEP' in lib.bsb_last_error()
  out.final_observation = None
  actions[3, 2] = -1                             # lane 2's budget is 0, but its mask is set: refused
  assert rollout(handle, T, actions.ctypes.data, 0, mask.ctypes.data, left.ctypes.data, ctypes.byref(out), None,
                 None) == 1
  actions[3, 2] = 0
  _lib.check(rollout(handle, T, actions.ctypes.data, 0, mask.ctypes.data, left.ctypes.data, ctypes.byref(out), None,
                     None))
  _lib.check(rollout(handle, T, None, 3, mask.ctypes.data, None, ctypes.byref(out), None, None))
  steps = ctypes.c_int64()
  _lib.check(lib.bsb_steps_done(handle, ctypes.byref(steps)))
  assert steps.value == 2 * T
  assert left.tolist() == [2, 2, 0]              # catch episodes are longer than 4 steps: no LAST yet
  assert not obs[:, 1].any()                     # lane 1 never made a call
  _lib.check(lib.bsb_destroy(handle))
