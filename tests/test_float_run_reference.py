"""`float_run_reference.expected_accumulators` pinned to the host path, bit for bit.

The host path (device='cpu') runs the same accumulator code as the kernels.  Here it runs whole float-dynamics runs --
complete default episodes, ~1 000 short episodes per lane so the log schedule reaches its later rows, mid-episode
resets, a same-step handle, a noise and a scale setting -- and `bsuite_info()`, `episode_stats()` and the log rows
must equal the model's, recomputed from the run's own rewards and step types.  The last tests show that the model
notices a float32 raw_return and a Logging restart at FIRST.
"""

import numpy as np
import pytest
import torch

import bsuite_b200
from bsuite_b200 import recording
from tests import float_run_reference as frr
from tests import float_step_reference as fr
from tests import gauss_draw_reference as gr

SEED = 7
SHORT = dict(cartpole=dict(max_time=.2), cartpole_swingup=dict(max_time=.2), mountain_car=dict(max_steps=9))


def _make(family, batch, rng='philox', params=None, noise_scale=None, reward_scale=None, **kw):
  kw = dict(dict(reward_dtype='float64', record_rows=True), **kw)
  return bsuite_b200.make(family, batch=batch, device='cpu', seed=SEED, rng=rng, noise_scale=noise_scale,
                          reward_scale=reward_scale, engine_kwargs=kw, **(params or {}))


def _run(env, T, chunk=1000, resets=(), twin=None, seed=0):
  """T calls of caller actions (rollouts of `chunk` calls; an explicit reset() at each call index in `resets`).
  Returns (rewards, step_types, unwrapped rewards of `twin` or None), each [T, B]."""
  actions = np.random.RandomState(seed).randint(0, env.num_actions, (T, env.batch)).astype(np.int32)
  rewards, types, unwrapped = [], [], []
  t = 0
  while t < T:
    if t in resets:
      ts = env.reset()
      rewards.append(np.zeros((1, env.batch)))
      types.append(ts.step_type.numpy()[None])
      if twin is not None:
        twin.reset()
        unwrapped.append(np.zeros((1, env.batch)))
      t += 1
      continue
    n = min([chunk, T - t] + [r - t for r in resets if r > t])
    a = torch.from_numpy(actions[t:t + n])
    ts = env.rollout(n, actions=a)
    rewards.append(ts.reward.numpy().astype(np.float64))
    types.append(ts.step_type.numpy())
    if twin is not None:
      unwrapped.append(twin.rollout(n, actions=a).reward.numpy())
    t += n
  cat = np.concatenate
  return cat(rewards), cat(types), (cat(unwrapped) if twin is not None else None)


def _assert_equal(label, env, acc):
  for name, got in env.bsuite_info().items():
    assert fr.mismatch(got.numpy(), acc.bsuite_info()[name]).sum() == 0, f'{label}: bsuite_info {name}'
  for name, got in env.episode_stats().items():
    bad = fr.mismatch(got.numpy(), acc.episode_stats()[name])
    assert not bad.any(), f'{label}: episode_stats {name} differs on {bad.sum()} lanes, first {np.flatnonzero(bad)[0]}'
  logged, want = env.logged_rows(), acc.logged_rows()
  assert np.array_equal(logged['counts'].numpy(), want['counts']), f'{label}: row counts'
  rows = logged['rows'].numpy()
  bad = np.flatnonzero(fr.mismatch(rows.transpose(2, 0, 1), want['rows'].transpose(2, 0, 1)))
  assert bad.size == 0, f'{label}: log rows differ on {bad.size} lanes, first {bad[0]}'


def _model(env, rewards, types, initial, unwrapped=None, **kw):
  return frr.expected_accumulators(frr.family_name(env), rewards, types, unwrapped, initial=initial,
                                   info_names=env.info_names, log_schedule=env.logged_rows()['schedule'],
                                   same_step=env.autoreset == 'same_step', **kw)


@pytest.mark.parametrize('rng', ['philox', 'mt19937'])
@pytest.mark.parametrize('family', fr.FAMILIES)
def test_complete_default_episodes(family, rng):
  env = _make(family, 8, rng)
  initial = frr.initial_state(env, env.state_dict()['blob'])
  rewards, types, _ = _run(env, 3000)
  assert (types == frr.LAST).sum(axis=0).min() >= 2
  _assert_equal(f'{family} {rng}', env, _model(env, rewards, types, initial))


@pytest.mark.parametrize('rng', ['philox', 'mt19937'])
@pytest.mark.parametrize('family', fr.FAMILIES)
def test_a_thousand_short_episodes(family, rng):
  env = _make(family, 6, rng, SHORT[family])
  initial = frr.initial_state(env, env.state_dict()['blob'])
  steps = 10 if family == 'mountain_car' else 22
  rewards, types, _ = _run(env, 1000 * steps + 50, chunk=4000)
  episodes = (types == frr.LAST).sum(axis=0)
  assert episodes.min() >= 1000, episodes
  assert env.logged_rows()['counts'].numpy().min() == len(recording.log_schedule(1000))
  _assert_equal(f'{family} short {rng}', env, _model(env, rewards, types, initial))


@pytest.mark.parametrize('family', fr.FAMILIES)
def test_mid_episode_resets(family):
  env = _make(family, 8, params=SHORT[family])
  initial = frr.initial_state(env, env.state_dict()['blob'])
  rewards, types, _ = _run(env, 400, chunk=7, resets=(0, 5, 6, 33, 100, 101, 250))
  _assert_equal(f'{family} resets', env, _model(env, rewards, types, initial))


@pytest.mark.parametrize('family', fr.FAMILIES)
def test_same_step_handle(family):
  env = _make(family, 8, params=SHORT[family], autoreset='same_step')
  initial = frr.initial_state(env, env.state_dict()['blob'])
  rewards, types, _ = _run(env, 600, chunk=9, resets=(0, 40, 41, 300))
  assert (types == frr.LAST).any() and not (types[1:] == frr.FIRST).all(axis=0).any()
  _assert_equal(f'{family} same_step', env, _model(env, rewards, types, initial))


@pytest.mark.parametrize('family,wrapper', [('cartpole', dict(noise_scale=.1)),
                                            ('mountain_car', dict(reward_scale=10.))])
def test_wrapped_rewards(family, wrapper):
  """Environment accumulators on the wrapper-free twin's reward, Logging columns on the wrapped reward."""
  env = _make(family, 8, params=SHORT[family], **wrapper)
  twin = gr.noise_free_twin(env)
  twin.load_state_dict(frr.transplant(env, env.state_dict()['blob'], twin))
  initial = frr.initial_state(env, env.state_dict()['blob'])
  rewards, types, unwrapped = _run(env, 2500, chunk=300, resets=(0, 77), twin=twin)
  assert not np.array_equal(rewards, unwrapped)
  _assert_equal(f'{family} {wrapper}', env, _model(env, rewards, types, initial, unwrapped))
  with pytest.raises(AssertionError):                # the unwrapped stream matters
    _assert_equal('wrapped only', env, _model(env, rewards, types, initial))


# ------------------------------------------------------------------ the model notices what it is there to catch
def test_a_float32_raw_return_changes_the_rows():
  env = _make('cartpole_swingup', 6, params=SHORT['cartpole_swingup'])
  initial = frr.initial_state(env, env.state_dict()['blob'])
  rewards, types, _ = _run(env, 3000, chunk=1000)
  good = _model(env, rewards, types, initial)
  bad = _model(env, rewards, types, initial, raw_dtype=np.float32)
  col = env.logged_rows()['columns'].index('raw_return')
  assert fr.mismatch(good.logged_rows()['rows'][:, col].T, bad.logged_rows()['rows'][:, col].T).all()
  with pytest.raises(AssertionError, match='bsuite_info raw_return'):
    _assert_equal('float32 raw_return', env, bad)


def test_a_restart_at_first_changes_the_rows():
  env = _make('cartpole', 6, params=SHORT['cartpole'])
  initial = frr.initial_state(env, env.state_dict()['blob'])
  rewards, types, _ = _run(env, 400, chunk=5, resets=(0, 3, 61, 62, 150))
  _assert_equal('restart after LAST', env, _model(env, rewards, types, initial))
  bad = _model(env, rewards, types, initial, restart='first')
  assert fr.mismatch(env.logged_rows()['rows'].numpy().transpose(2, 0, 1),
                     bad.logged_rows()['rows'].transpose(2, 0, 1)).any()
  with pytest.raises(AssertionError):
    _assert_equal('restart at FIRST', env, bad)


def test_run_script_is_reproducible_and_covers_the_calls():
  a = frr.run_script(101, 33, 3, seed=4, masks=True, budgets=True)
  b = frr.run_script(101, 33, 3, seed=4, masks=True, budgets=True)
  assert np.array_equal(a['actions'], b['actions']) and np.array_equal(a['budgets'], b['budgets'])
  assert sum(n for _, n, _ in a['segments']) == 101
  assert {k for k, _, _ in a['segments']} == {'rollout', 'step'}
  assert all(np.array_equal(x[2], y[2]) for x, y in zip(a['segments'], b['segments']))
  assert a['budgets'].min() >= 0 and a['budgets'].max() <= 3
