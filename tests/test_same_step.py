"""Same-step auto-reset (`autoreset='same_step'`, BSB_FLAG_SAME_STEP_RESET) on the explicit host path.

Under same-step, lane i's outputs are the reference's own call sequence for that lane with every LAST call merged
into the reset call that follows it.  So the golden fixtures check it directly: drop each call that follows a LAST
(and its ignored action), take that call's FIRST observation as the merged call's `observation` and the LAST's
observation as its `final_observation`.  The next-step host path, pinned to the reference by the golden and oracle
tests, checks the rest over long runs: info, Logging columns and log rows included.
"""

import ctypes
import itertools

import numpy as np
import pytest
import torch

import bsuite_b200
from bsuite_b200 import _lib
from bsuite_b200 import sweep
from tests import conftest as cf

SENTINEL = 7.0      # written into final_observation before every call: rows of lanes that did not finish keep it


def _make(meta, lane, autoreset, final=True):
  kwargs = dict(meta['kwargs'])
  wrap = {}
  if meta['wrapper'] == 'noise':
    wrap['noise_scale'] = meta['wrapper_arg']
  elif meta['wrapper'] == 'scale':
    wrap['reward_scale'] = meta['wrapper_arg']
  return bsuite_b200.make(meta['env_class'], batch=1, device='cpu', seed=meta['seed'], rng=meta['rng'],
                          engine_kwargs=dict(reward_dtype='float64', autoreset=autoreset, lane_offset=lane),
                          **wrap, **kwargs)


def fold(step_type, reset_at):
  """The calls of one lane under same-step: (kind, reference call, reference call whose observation it returns).

  kind 'reset' is an explicit reset() (FIRST); 'step' a transition.  A transition that returned LAST is merged with
  the reference's next call -- the automatic reset, or an explicit reset() made right after the LAST, which resets
  the lane once all the same -- and returns that call's observation.  When the trace ends on LAST, that observation
  is not in the fixture (None): the call is still made, for its other outputs and for bsuite_info()."""
  calls, t, T = [], 0, len(step_type)
  while t < T:
    if t in reset_at:
      calls.append(('reset', t, t))
      t += 1
      continue
    if step_type[t] == 2:
      calls.append(('step', t, t + 1 if t + 1 < T else None))
      t += 2
      continue
    calls.append(('step', t, t))
    t += 1
  return calls


def test_fold_of_a_short_trace():
  #            F  M  L  F  M  L  F  L
  st = np.array([0, 1, 2, 0, 1, 2, 0, 2])
  assert fold(st, set()) == [('step', 0, 0), ('step', 1, 1), ('step', 2, 3), ('step', 4, 4), ('step', 5, 6),
                             ('step', 7, None)]
  assert fold(st, {4}) == [('step', 0, 0), ('step', 1, 1), ('step', 2, 3), ('reset', 4, 4), ('step', 5, 6),
                           ('step', 7, None)]


PHILOX_CASES = [n for n in cf.golden_case_names() if cf.load_golden(n)[0]['rng'] == 'philox']
MT_CASES = [n for n in cf.golden_case_names() if cf.load_golden(n)[0]['rng'] != 'philox']


def _make_on(meta, lane, device):
  kwargs = dict(meta['kwargs'])
  wrap = {}
  if meta['wrapper'] == 'noise':
    wrap['noise_scale'] = meta['wrapper_arg']
  elif meta['wrapper'] == 'scale':
    wrap['reward_scale'] = meta['wrapper_arg']
  return bsuite_b200.make(meta['env_class'], batch=1, device=device, seed=meta['seed'], rng=meta['rng'],
                          engine_kwargs=dict(reward_dtype='float64', autoreset='same_step', lane_offset=lane),
                          **wrap, **kwargs)


def run_folded_lane(meta, data, k, device='cpu', fused=False):
  """Lane k of a fixture as a one-lane same-step handle at lane_offset = its lane, driven through its folded calls.

  Stepwise: one step() / reset() per folded call.  Fused: the steps between explicit resets as one rollout each.
  `final_observation` is filled with SENTINEL before every call.  Returns (calls, outputs stacked over the calls,
  bsuite_info)."""
  calls = fold(data['step_type'][:, k], set(meta['reset_at']))
  env = _make_on(meta, meta['lanes'][k], device)
  fields = ('step_type', 'reward', 'discount', 'observation', 'final_observation')
  res = {f: [] for f in fields}
  try:
    c = 0
    while c < len(calls):
      kind, t, _ = calls[c]
      if kind == 'reset' or not fused:
        out = env.make_buffers(final_observation=True)
        out.final_observation.fill_(SENTINEL)
        if kind == 'reset':
          env.reset(out=out)
        else:
          env.step(torch.tensor([data['actions'][t, k]], dtype=torch.int32, device=env.device), out=out)
        for f in fields:
          res[f].append(getattr(out, f).cpu().numpy().copy())
        c += 1
        continue
      run = c
      while run < len(calls) and calls[run][0] == 'step':
        run += 1
      acts = np.array([[data['actions'][calls[j][1], k]] for j in range(c, run)], np.int32)
      out = env.make_buffers(run - c, final_observation=True)
      out.final_observation.fill_(SENTINEL)
      env.rollout(run - c, actions=torch.as_tensor(acts, device=env.device), out=out)
      for f in fields:
        res[f].extend(getattr(out, f).cpu().numpy().copy())
      c = run
    info = {key: float(v.cpu()[0]) for key, v in env.bsuite_info().items()}
  finally:
    env.close()
  return calls, {f: np.stack(v) for f, v in res.items()}, info


def check_folded_lane(name, meta, data, k, calls, res, info, reward_tol=0.0, obs_tol=0.0):
  """The folded outputs of lane k against the fixture: every reference value exactly once.  `reward_tol` is a number
  or a function of the reward returned."""
  obs_shape = data['observation'].shape[2:]
  close = lambda got, want, where, tol: np.testing.assert_allclose(got, want, rtol=0, atol=tol, err_msg=where) if tol \
      else np.testing.assert_array_equal(got, want, err_msg=where)
  for c, (kind, t, t_obs) in enumerate(calls):
    where = f'{name} lane {meta["lanes"][k]} reference call {t} ({kind})'
    st = data['step_type'][t, k]
    assert res['step_type'][c].reshape(-1)[0] == st, where
    if t_obs is not None:
      close(res['observation'][c].reshape(obs_shape), data['observation'][t_obs, k].reshape(obs_shape), where, obs_tol)
    if st == 0:
      assert res['reward'][c].reshape(-1)[0] == 0.0 and res['discount'][c].reshape(-1)[0] == 0.0, where
    else:
      got = res['reward'][c].reshape(-1)[0]
      close(got, data['reward'][t, k], where + ' reward', reward_tol(got) if callable(reward_tol) else reward_tol)
      assert res['discount'][c].reshape(-1)[0] == data['discount'][t, k], where
    final = res['final_observation'][c].reshape(obs_shape)
    if st == 2:
      close(final, data['observation'][t, k].reshape(obs_shape), where + ' final_observation', obs_tol)
    else:
      assert np.all(final == SENTINEL), where + ': final_observation written for a lane that did not finish'
  for j, key in enumerate(meta['info_names']):
    want = data['info'][k, j]
    tol = 0.0 if not (reward_tol or obs_tol) else 1e-6 * max(1.0, abs(want))
    assert abs(info[key] - want) <= tol, f'{name} lane {meta["lanes"][k]} bsuite_info[{key}]: {info[key]} != {want}'


@pytest.mark.parametrize('fused', [False, True], ids=['stepwise', 'fused'])
@pytest.mark.parametrize('name', PHILOX_CASES)
def test_host_path_folds_the_reference_trace(name, fused, mnist_dir):
  """Bit for bit, float families included (the host path calls libm as numpy does)."""
  meta, data = cf.load_golden(name)
  for k in range(len(meta['lanes'])):
    calls, res, info = run_folded_lane(meta, data, k, 'cpu', fused)
    check_folded_lane(name, meta, data, k, calls, res, info)


@pytest.mark.parametrize('name', MT_CASES)
def test_mt19937_is_refused(name):
  meta, _ = cf.load_golden(name)
  with pytest.raises(_lib.EngineError, match='status 2'):
    _make(meta, 0, 'same_step')


# ------------------------------------------------------------------ against the next-step host path
def _experiment_ids():
  return [sweep.BY_EXPERIMENT[name][0] for name in sweep.BY_EXPERIMENT]


def _twin_case(bsuite_id):
  # long episodes (cartpole: up to 1 000 steps) are capped by calls rather than episodes
  return dict(episodes=300, max_calls=2500, lanes=(0, 5))


@pytest.mark.parametrize('bsuite_id', _experiment_ids())
def test_same_step_is_the_folded_next_step_trace(bsuite_id, mnist_dir):
  case = _twin_case(bsuite_id)
  for lane in case['lanes']:
    same = bsuite_b200.load_from_id(bsuite_id, batch=1, device='cpu', seed=11, lane_offset=lane, record_rows=True,
                                    reward_dtype='float64', autoreset='same_step')
    nxt = bsuite_b200.load_from_id(bsuite_id, batch=1, device='cpu', seed=11, lane_offset=lane, record_rows=True,
                                   reward_dtype='float64')
    try:
      _drive_pair(bsuite_id, lane, same, nxt, case)
    finally:
      same.close()
      nxt.close()


def _snapshot(env, out):
  return {f: getattr(out, f).numpy().copy() for f in ('step_type', 'reward', 'discount', 'observation')}


def _drive_pair(bsuite_id, lane, same, nxt, case):
  rng = np.random.RandomState(lane + 3)
  so = same.make_buffers(final_observation=True)
  no = nxt.make_buffers()
  episodes, calls = 0, 0
  act = lambda a: torch.tensor([a], dtype=torch.int32)
  # the first call of both handles: FIRST
  a = int(rng.randint(same.num_actions))
  same.step(act(a), out=so)
  nxt.step(act(a), out=no)
  s, n = _snapshot(same, so), _snapshot(nxt, no)
  for f in s:
    np.testing.assert_array_equal(s[f], n[f], err_msg=f'{bsuite_id} lane {lane} first call {f}')
  while episodes < case['episodes'] and calls < case['max_calls']:
    calls += 1
    a = int(rng.randint(same.num_actions))
    so.final_observation.fill_(SENTINEL)
    same.step(act(a), out=so)
    nxt.step(act(a), out=no)
    s, n = _snapshot(same, so), _snapshot(nxt, no)
    where = f'{bsuite_id} lane {lane} call {calls}'
    for f in ('step_type', 'reward', 'discount'):
      np.testing.assert_array_equal(s[f], n[f], err_msg=f'{where} {f}')
    if n['step_type'][0] == 2:
      episodes += 1
      np.testing.assert_array_equal(so.final_observation.numpy(), n['observation'], err_msg=f'{where} final_observation')
      if episodes % 50 == 1:      # the Logging columns at the LAST, before the next-step twin's reset call
        _compare_stats(where, same, nxt)
      nxt.step(act(int(rng.randint(same.num_actions))), out=no)      # the next-step twin's reset call
      assert int(no.step_type[0]) == 0, where
      np.testing.assert_array_equal(s['observation'], no.observation.numpy(), err_msg=f'{where} observation')
    else:
      np.testing.assert_array_equal(s['observation'], n['observation'], err_msg=f'{where} observation')
      assert np.all(so.final_observation.numpy() == SENTINEL), where
  assert episodes >= min(case['episodes'], 2), f'{bsuite_id}: only {episodes} episodes'
  where = f'{bsuite_id} lane {lane} end'
  for key, value in same.bsuite_info().items():
    np.testing.assert_array_equal(value.numpy(), nxt.bsuite_info()[key].numpy(), err_msg=f'{where} {key}')
  got, want = same.logged_rows(), nxt.logged_rows()
  np.testing.assert_array_equal(got['counts'].numpy(), want['counts'].numpy(), err_msg=f'{where} log row counts')
  np.testing.assert_array_equal(got['rows'].numpy(), want['rows'].numpy(), err_msg=f'{where} log rows')
  # one more transition on both: the columns restart on the same-step handle's next call too
  a = int(rng.randint(same.num_actions))
  same.step(act(a), out=so)
  nxt.step(act(a), out=no)
  _compare_stats(where + ' +1', same, nxt)


def _compare_stats(where, same, nxt):
  got, want = same.episode_stats(), nxt.episode_stats()
  for key in ('episode', 'total_return', 'episode_len', 'episode_return'):
    np.testing.assert_array_equal(got[key].numpy(), want[key].numpy(), err_msg=f'{where} episode_stats[{key}]')
  # `steps` counts transitions: the next-step twin's extra calls are all FIRST
  assert float(got['steps'][0]) == float(want['steps'][0]), f'{where} episode_stats[steps]'


def test_explicit_reset_restarts_the_logging_columns(mnist_dir):
  """A reset() right after a merged reset, and one in the middle of an episode, against the next-step twin."""
  same = bsuite_b200.load_from_id('catch/0', batch=1, device='cpu', seed=3, track_episodes=True, autoreset='same_step')
  nxt = bsuite_b200.load_from_id('catch/0', batch=1, device='cpu', seed=3, track_episodes=True)
  one = torch.ones(1, dtype=torch.int32)
  try:
    same.step(one)
    nxt.step(one)
    for _ in range(9):           # catch/0: 9 transitions per episode, the 9th merged with the reset
      same.step(one)
      nxt.step(one)
    _compare_stats('after LAST', same, nxt)
    same.reset()
    nxt.step(one)                # the twin's automatic reset ...
    _compare_stats('after the reset (same-step) / automatic reset (next-step)', same, nxt)
    for _ in range(4):
      same.step(one)
      nxt.step(one)
      _compare_stats('mid-episode', same, nxt)
  finally:
    same.close()
    nxt.close()


# ------------------------------------------------------------------ snapshots and arguments
def test_snapshots_keep_their_mode():
  a = bsuite_b200.load_from_id('deep_sea/0', batch=4, device='cpu', seed=1, track_episodes=True)
  b = bsuite_b200.load_from_id('deep_sea/0', batch=4, device='cpu', seed=1, track_episodes=True)
  c = bsuite_b200.load_from_id('deep_sea/0', batch=4, device='cpu', seed=1, track_episodes=True, autoreset='same_step')
  d = bsuite_b200.load_from_id('deep_sea/0', batch=4, device='cpu', seed=1, track_episodes=True, autoreset='same_step')
  try:
    a.rollout(7, action_seed=2)
    b.load_state_dict(a.state_dict())          # next-step into next-step, as before
    np.testing.assert_array_equal(a.rollout(30, action_seed=3).observation.numpy(),
                                  b.rollout(30, action_seed=3).observation.numpy())
    with pytest.raises(ValueError):
      c.load_state_dict(a.state_dict())
    with pytest.raises(ValueError):
      a.load_state_dict(c.state_dict())
    c.rollout(25, action_seed=2)
    d.load_state_dict(c.state_dict())
    oc, od = c.make_buffers(9, final_observation=True), d.make_buffers(9, final_observation=True)
    c.rollout(9, action_seed=4, out=oc)
    d.rollout(9, action_seed=4, out=od)
    for f in ('observation', 'final_observation', 'step_type', 'reward'):
      np.testing.assert_array_equal(getattr(oc, f).numpy(), getattr(od, f).numpy(), err_msg=f)
    for k in c.episode_stats():
      np.testing.assert_array_equal(c.episode_stats()[k].numpy(), d.episode_stats()[k].numpy(), err_msg=k)
  finally:
    for env in (a, b, c, d):
      env.close()


def _config(rng_kind, flags):
  cfg = _lib.Config()
  cfg.family, cfg.rng_kind, cfg.flags = _lib.CATCH, rng_kind, flags
  cfg.rows, cfg.columns, cfg.deterministic, cfg.reward_scale = 10, 5, 1, 1.0
  return cfg


def test_argument_checks():
  lib = _lib.load()
  env = ctypes.c_void_p()
  assert lib.bsb_create(ctypes.byref(_config(_lib.RNG_MT19937, _lib.FLAG_SAME_STEP_RESET)), 4, _lib.DEVICE_HOST, 1, 0,
                        ctypes.byref(env)) == 2
  assert b'PHILOX' in lib.bsb_last_error()
  obs = np.zeros((4, 50), np.float32)
  final = np.zeros((4, 50), np.float32)
  actions = np.zeros(4, np.int32)
  out = _lib.Outputs(observation=obs.ctypes.data, final_observation=final.ctypes.data)
  for flags, want_step, want_host in ((0, 1, 2), (_lib.FLAG_SAME_STEP_RESET, 0, 2)):
    assert lib.bsb_create(ctypes.byref(_config(_lib.RNG_PHILOX, flags)), 4, _lib.DEVICE_HOST, 1, 0, ctypes.byref(env)) == 0
    try:
      assert lib.bsb_reset(env, ctypes.byref(out), None) == want_step
      assert lib.bsb_step(env, actions.ctypes.data, ctypes.byref(out), None) == want_step
      assert lib.bsb_rollout(env, 1, actions.ctypes.data, 0, ctypes.byref(out), None, None) == want_step
      assert lib.bsb_step_host(env, actions.ctypes.data, ctypes.byref(out), None, None, 0) == want_host
    finally:
      lib.bsb_destroy(env)


def test_python_argument_checks():
  with pytest.raises(ValueError, match='autoreset'):
    bsuite_b200.load_from_id('catch/0', autoreset='same_step', device='cpu')          # the B = 1 face
  with pytest.raises(ValueError, match='autoreset'):
    bsuite_b200.load_from_id('catch/0', batch=2, device='cpu', autoreset='disabled')
  with pytest.raises(_lib.EngineError):
    bsuite_b200.load_from_id('catch/0', batch=2, device='cpu', rng='mt19937', autoreset='same_step')
  env = bsuite_b200.load_from_id('catch/0', batch=2, device='cpu')
  with pytest.raises(ValueError, match='final_observation'):
    env.make_buffers(final_observation=True)
  env.close()
  env = bsuite_b200.load_from_id('catch/0', batch=2, device='cpu', autoreset='same_step', obs_dtype='bfloat16')
  out = env.make_buffers(final_observation=True)
  out.final_observation = out.final_observation.float()
  with pytest.raises(ValueError, match='final_observation'):
    env.step(torch.zeros(2, dtype=torch.int32), out=out)
  env.close()


def test_sweep_batch_forwards_the_mode(mnist_dir):
  from bsuite_b200.suite import SweepBatch
  batch = SweepBatch(['bandit/0', 'catch/0'], lanes=8, device='cpu', autoreset='same_step')
  assert {env.autoreset for env in batch.envs.values()} == {'same_step'}


def test_collect_and_replay_use_the_final_observation():
  from bsuite_b200 import rollouts
  env = bsuite_b200.load_from_id('catch/0', batch=3, device='cpu', seed=2, autoreset='same_step')
  trajectory, finals = rollouts.collect(env, 25, action_seed=1, final_observations=True)
  replay = rollouts.Replay(1000, device='cpu')
  n = replay.add_transitions(trajectory, finals)
  assert n == int((trajectory.step_types != 0).sum())
  o_t = replay._data[4][:n]
  d_t = replay._data[3][:n]
  keep = (trajectory.step_types != 0).reshape(-1)
  last = (trajectory.step_types == 2).reshape(-1)[keep]
  np.testing.assert_array_equal(o_t[last].numpy(), finals.reshape((-1,) + finals.shape[2:])[(trajectory.step_types == 2).reshape(-1)].numpy())
  assert bool((d_t[last] == 0).all())
  # the LAST boards of catch show the ball on the bottom row, the next episode's first boards show it on the top
  assert float(finals[trajectory.step_types == 2][:, :-1].sum()) == 0.0
  assert bool((trajectory.observations[1:][trajectory.step_types == 2][:, 0].sum(-1) == 1).all())
  env.close()


# ------------------------------------------------------------------ coverage of the GPU file
def test_gpu_cases_cover_every_same_step_instantiation():
  from bsuite_b200 import build
  from tests import test_same_step_gpu as g
  want = set()
  for family in cf_families():
    dtypes = ('float32', 'bfloat16') + (('uint8',) if family in ('deep_sea', 'catch') else ())
    for dtype, noise, track in itertools.product(dtypes, (False, True), (False, True)):
      want.add((family, dtype, noise, track))
  got = {(c['family'], c['obs_dtype'], c['noise'] is not None, bool(c['track'])) for c in g.GROUP_S}
  assert len(want) == 88
  names = {'float': 'float32', 'Bf16': 'bfloat16', 'uint8_t': 'uint8'}
  units = {unit[3:]: rows for unit, rows in build.variant_list().items() if unit.startswith('ss_')}
  assert all(mode == 'SAME_STEP' and not mt and not tp for rows in units.values() for _, _, mode, mt, tp in rows)
  assert {(f, names[o]) for f, rows in units.items() for _, o, _, _, _ in rows} == {w[:2] for w in want}
  assert want <= got, sorted(want - got)


def cf_families():
  from bsuite_b200 import build
  return build.FAMILIES
