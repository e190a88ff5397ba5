"""One CUDA step of cartpole, cartpole_swingup and mountain_car against the one-step envelope, to the ulp.

Every device test elsewhere compares whole float-family trajectories within FLOAT_TOL (1e-6), which measures
accumulated drift, not the step.  Here every lane is resynchronised: the same state is injected into a CUDA handle
and a device='cpu' twin through the state_dict() blob (tests/float_step_reference.py: inject_states), both take ONE
step, and per lane:

  * outputs that read no trig (x, theta, t, tick and the observation entries made from them) equal the host's bit
    for bit;
  * x_dot, theta_dot, vel, pos and the observation lie in the device envelope (CUDA's double sin / cos / sincos
    within TRIG_ULPS = 2 ulp of the correctly rounded value, every other operation IEEE in the reference's order);
  * step type, discount, reward and bsuite_info() equal the host's, and step type, discount and reward equal the
    reference step's, wherever every decision is robust in the envelope (elsewhere either outcome is a correct step;
    the count is printed).

Trig lanes (theta_dot = 0 or vel = 0, action 1) measure the device's trig error directly: the smallest ulp offsets
from the correctly rounded sin / cos that reproduce the new velocities are printed.  Then every kernel a float family
goes through runs once on a subset of the states: single steps at B = 4099 with Philox and MT19937, with and without
episode tracking, rollout(1), a masked step, a same-step handle, the packed cartpole_swingup experiment and a bfloat16
handle.
"""

import numpy as np
import pytest
import torch

import bsuite_b200
from bsuite_b200 import sweep
from tests import float_step_reference as fr

pytestmark = pytest.mark.gpu

SUBSET = 4099                  # 128 full 32-lane chunks and a 3-lane tail
SEED = 11


def _make(family, batch, device, **kw):
  kw.setdefault('reward_dtype', 'float64')
  rng = kw.pop('rng', 'philox')
  return bsuite_b200.make(family, batch=batch, device=device, seed=SEED, rng=rng, engine_kwargs=kw)


def _inject_pair(dev, host, states):
  """The same blob (built from the CUDA handle's own snapshot) into both handles."""
  dev.reset()
  torch.cuda.synchronize()
  sd = fr.inject_states(dev, states)
  dev.load_state_dict(sd)
  host.load_state_dict(sd)           # the config fingerprint does not include the device


def _outputs(env, ts, n, final=None):
  out = dict(step_type=ts.step_type.cpu().numpy().reshape(n), discount=ts.discount.cpu().numpy().reshape(n),
             reward=ts.reward.cpu().numpy().reshape(n), obs=ts.observation.float().cpu().numpy().reshape(n, -1),
             state=fr.read_states(env), info={k: v.cpu().numpy() for k, v in env.bsuite_info().items()})
  if final is not None:
    out['final_obs'] = final.float().cpu().numpy().reshape(n, -1)
  return out


def _bits_equal(a, b):
  return ~fr.mismatch(a, b)


def _round_obs(dtype):
  if dtype == 'bfloat16':
    return lambda a: torch.from_numpy(np.ascontiguousarray(a, np.float32)).to(torch.bfloat16).float().numpy()
  return lambda a: a


def _check(label, family, env, gpu, host, lanes=None, obs_dtype='float32', obs_key='obs', state=True):
  """The assertions of the module docstring on `lanes` (default all) of one step; returns the non-robust count.
  `state=False`: lanes that have started a new episode since (same-step auto-reset), whose state is not the step's."""
  n = gpu['step_type'].shape[0]
  lanes = np.arange(n) if lanes is None else np.asarray(lanes)
  robust = env['robust'][lanes]
  sel = lambda a: np.asarray(a)[lanes]
  for f in fr.EXACT_STATE[family] if state else ():
    bad = ~_bits_equal(sel(gpu['state'][f]), sel(host['state'][f]))
    assert not bad.any(), f'{label}: {f} is not bit-exact on {bad.sum()} lanes, first lane {lanes[bad][0]}'
  for f in fr.ENVELOPE_STATE[family] if state else ():
    bad = fr.outside(sel(env['lo'][f]), sel(env['hi'][f]), sel(gpu['state'][f]))
    assert not bad.any(), (f'{label}: {f} outside the envelope on {bad.sum()} lanes, first lane {lanes[bad][0]}: '
                           f'{sel(gpu["state"][f])[bad][0]!r} not in [{sel(env["lo"][f])[bad][0]!r}, '
                           f'{sel(env["hi"][f])[bad][0]!r}]')
  rnd = _round_obs(obs_dtype)
  obs, hobs = sel(gpu[obs_key]), sel(host[obs_key])
  for col in fr.EXACT_OBS[family]:
    bad = ~_bits_equal(obs[:, col], hobs[:, col])
    assert not bad.any(), f'{label}: observation column {col} is not bit-exact on {bad.sum()} lanes'
  bad = fr.outside(rnd(sel(env['lo']['obs'])), rnd(sel(env['hi']['obs'])), obs).any(axis=1)
  assert not bad.any(), (f'{label}: observation outside the envelope on {bad.sum()} lanes, first lane '
                         f'{lanes[bad][0]}: {obs[bad][0]} vs host {hobs[bad][0]}')
  for f in ('step_type', 'discount', 'reward'):
    bad = robust & ~_bits_equal(sel(gpu[f]), sel(host[f]))
    assert not bad.any(), f'{label}: {f} differs from the host on {bad.sum()} robust lanes, first {lanes[bad][0]}'
    bad = robust & ~_bits_equal(sel(gpu[f]), sel(env['center'][f]))
    assert not bad.any(), (f'{label}: {f} differs from the reference step on {bad.sum()} robust lanes, first '
                           f'{lanes[bad][0]}')
  for f, v in gpu['info'].items():
    bad = robust & ~_bits_equal(sel(v), sel(host['info'][f]))
    assert not bad.any(), f'{label}: bsuite_info {f} differs on {bad.sum()} robust lanes, first {lanes[bad][0]}'
  if family != 'mountain_car' and state:
    bad = robust & ~_bits_equal(sel(gpu['state']['episode_return']), sel(host['state']['episode_return']))
    assert not bad.any(), f'{label}: episode_return differs on {bad.sum()} robust lanes'
  return int((~robust).sum())


def _trig_error(family, params, states, actions, kind, gpu, max_ulps=8):
  """On the trig lanes with action 1: the smallest |ulp offsets| of (sin, cos) from the correctly rounded values that
  reproduce the device's new velocities; returns (largest sin offset, largest cos offset, lanes no offset explains)."""
  lanes = np.flatnonzero((kind == 1) & (actions == 1))
  st, act = fr.select(states, lanes), actions[lanes]
  fields = ('vel',) if family == 'mountain_car' else ('x_dot', 'theta_dot')
  got = [gpu['state'][f][lanes] for f in fields]
  best = np.full((lanes.size, 2), max_ulps + 1)
  table = fr._TrigTable()                                     # pylint: disable=protected-access
  sins = [0] if family == 'mountain_car' else range(-max_ulps, max_ulps + 1)
  for i in sins:
    for j in range(-max_ulps, max_ulps + 1):
      run = fr.offset_step(family, params, st, act, (i, j), table)
      hit = np.all([_bits_equal(run['state'][f], g) for f, g in zip(fields, got)], axis=0)
      better = hit & (max(abs(i), abs(j)) < best.max(axis=1))
      best[better] = (abs(i), abs(j))
  unexplained = int((best.max(axis=1) > max_ulps).sum())
  found = best[best.max(axis=1) <= max_ulps]
  return (int(found[:, 0].max()) if found.size else -1, int(found[:, 1].max()) if found.size else -1, unexplained)


@pytest.mark.parametrize('family', fr.FAMILIES)
def test_one_device_step_lies_in_the_envelope(family):
  params, states, actions, kind = fr.cached_case(family)
  env = fr.cached_envelope(family)
  n = actions.shape[0]
  dev, host = _make(family, n, 'cuda'), _make(family, n, 'cpu')
  _inject_pair(dev, host, states)
  act = torch.from_numpy(actions)
  gpu = _outputs(dev, dev.step(act.cuda()), n)
  cpu = _outputs(host, host.step(act), n)
  non_robust = _check(family, family, env, gpu, cpu)
  sin_ulp, cos_ulp, unexplained = _trig_error(family, params, states, actions, kind, gpu)
  trig = f'cos <= {cos_ulp} ulp' if family == 'mountain_car' else f'sin <= {sin_ulp} ulp, cos <= {cos_ulp} ulp'
  print(f'\n[float step] {family}: {n} lanes, {non_robust} with a non-robust decision; device trig error on '
        f'{int(((kind == 1) & (actions == 1)).sum())} trig lanes: {trig} ({unexplained} lanes unexplained within '
        '8 ulp)')
  assert unexplained == 0


# ------------------------------------------------------------------ launch paths
def _subset(family):
  params, states, actions, kind = fr.cached_case(family)
  lanes = np.concatenate([np.flatnonzero(kind == 0), np.flatnonzero(kind == 1)[:64], np.flatnonzero(kind == 2)])
  lanes = lanes[:SUBSET]
  return params, fr.select(states, lanes), actions[lanes], lanes


PLAIN = [('philox', False), ('mt19937', False), ('philox', True), ('mt19937', True)]


@pytest.mark.parametrize('rng,track', PLAIN, ids=['philox', 'mt19937', 'philox-track', 'mt19937-track'])
@pytest.mark.parametrize('family', fr.FAMILIES)
def test_single_step_paths(family, rng, track):
  params, states, actions, lanes = _subset(family)
  env = fr.device_envelope(family, params, states, actions)
  n = actions.shape[0]
  dev, host = _make(family, n, 'cuda', rng=rng, track_episodes=track), _make(family, n, 'cpu', rng=rng,
                                                                              track_episodes=track)
  _inject_pair(dev, host, states)
  act = torch.from_numpy(actions)
  gpu, cpu = _outputs(dev, dev.step(act.cuda()), n), _outputs(host, host.step(act), n)
  _check(f'{family} {rng} track={track}', family, env, gpu, cpu)
  if track:
    robust = env['robust']
    for f, v in dev.episode_stats().items():
      assert np.array_equal(v.cpu().numpy()[robust], host.episode_stats()[f].numpy()[robust]), f


@pytest.mark.parametrize('family', fr.FAMILIES)
def test_rollout_of_one_step(family):
  params, states, actions, _ = _subset(family)
  env = fr.device_envelope(family, params, states, actions)
  n = actions.shape[0]
  dev, host = _make(family, n, 'cuda'), _make(family, n, 'cpu')
  _inject_pair(dev, host, states)
  act = torch.from_numpy(actions)[None]
  gpu, cpu = _outputs(dev, dev.rollout(1, actions=act.cuda()), n), _outputs(host, host.rollout(1, actions=act), n)
  _check(f'{family} rollout(1)', family, env, gpu, cpu)


@pytest.mark.parametrize('family', fr.FAMILIES)
def test_masked_step(family):
  params, states, actions, _ = _subset(family)
  env = fr.device_envelope(family, params, states, actions)
  n = actions.shape[0]
  dev, host = _make(family, n, 'cuda'), _make(family, n, 'cpu')
  _inject_pair(dev, host, states)
  mask = np.arange(n) % 2 == 0
  act = torch.from_numpy(actions)
  dout, hout = dev.make_buffers(), host.make_buffers()
  gpu = _outputs(dev, dev.step(act.cuda(), out=dout, mask=torch.from_numpy(mask).cuda()), n)
  cpu = _outputs(host, host.step(act, out=hout, mask=torch.from_numpy(mask)), n)
  _check(f'{family} masked', family, env, gpu, cpu, lanes=np.flatnonzero(mask))
  off = ~mask
  for f in fr.STATE_FIELDS[family]:
    want = np.asarray(states[f], gpu['state'][f].dtype)
    assert _bits_equal(gpu['state'][f][off], want[off]).all(), f'masked-off lanes changed {f}'
  assert not gpu['state']['needs_reset'][off].any()


def _reset_obs_envelope(family, params, st):
  """[lo, hi] of the first observation of a freshly reset state (exact but for the pole's sin / cos entries)."""
  if family == 'mountain_car':
    o = np.stack([st['pos'], st['vel'], st['tick'] / params['max_steps']], axis=1).astype(np.float32)
    return o, o
  x_thr = params['x_threshold']
  rows = []
  for d in (-fr.TRIG_ULPS, fr.TRIG_ULPS):
    r = [st['x'] / x_thr, st['x_dot'] / x_thr, fr.nudge(fr.correctly_rounded('sin', st['theta']), d),
         fr.nudge(fr.correctly_rounded('cos', st['theta']), d), st['theta_dot'], st['t'] / params['max_time']]
    if family == 'cartpole_swingup':
      r += [np.where(np.abs(st['x']) < params['x_reward_threshold'], 1., -1.),
            np.where(np.abs(st['theta_dot']) < params['theta_dot_threshold'], 1., -1.)]
    rows.append(np.stack(r, axis=1).astype(np.float32))
  return rows[0], rows[1]


@pytest.mark.parametrize('family', fr.FAMILIES)
def test_same_step_handle(family):
  params, states, actions, _ = _subset(family)
  env = fr.device_envelope(family, params, states, actions)
  n = actions.shape[0]
  dev, host = _make(family, n, 'cuda', autoreset='same_step'), _make(family, n, 'cpu', autoreset='same_step')
  _inject_pair(dev, host, states)
  act = torch.from_numpy(actions)
  dout, hout = dev.make_buffers(final_observation=True), host.make_buffers(final_observation=True)
  gpu = _outputs(dev, dev.step(act.cuda(), out=dout), n, final=dout.final_observation)
  cpu = _outputs(host, host.step(act, out=hout), n, final=hout.final_observation)
  robust = env['robust']
  last = robust & (cpu['step_type'] == fr.LAST)
  mid = robust & (cpu['step_type'] == fr.MID)
  assert last.any() and mid.any()
  _check(f'{family} same_step', family, env, gpu, cpu, lanes=np.flatnonzero(mid))
  _check(f'{family} same_step final', family, env, gpu, cpu, lanes=np.flatnonzero(last), obs_key='final_obs',
         state=False)
  # lanes that finished start their next episode in the same call: the reset draws are exact
  for f in fr.STATE_FIELDS[family]:
    assert _bits_equal(gpu['state'][f][last], cpu['state'][f][last]).all(), f'reset {f}'
  lo, hi = _reset_obs_envelope(family, params, fr.select(cpu['state'], last))
  assert not fr.outside(lo, hi, gpu['obs'][last]).any()


def test_packed_cartpole_swingup():
  """All 20 settings of cartpole_swingup in one environment, each setting's lanes holding the edge states built for
  its own height_threshold and x_reward_threshold."""
  ids = sweep.BY_EXPERIMENT['cartpole_swingup']
  per = {}
  for bsuite_id in ids:
    params = fr.default_params('cartpole_swingup', **sweep.SETTINGS[bsuite_id])
    states, actions, _ = fr.build_states('cartpole_swingup', params, n_random=0, n_trig=0, seed=1)
    per[bsuite_id] = (params, states, actions)
  lanes = min(a.shape[0] for _, _, a in per.values())
  dev = bsuite_b200.load_experiment('cartpole_swingup', lanes, device='cuda', seed=SEED, reward_dtype='float64')
  host = bsuite_b200.load_experiment('cartpole_swingup', lanes, device='cpu', seed=SEED, reward_dtype='float64')
  n = dev.batch
  per = {i: (p, fr.select(s, slice(0, lanes)), a[:lanes]) for i, (p, s, a) in per.items()}
  # each setting's states go into the lanes the pack gives that setting
  states = {k: np.zeros(n, v.dtype) for k, v in per[ids[0]][1].items()}
  actions = np.zeros(n, np.int32)
  filled = np.zeros(n, np.int32)
  for bsuite_id, (_, s, a) in per.items():
    sl = dev.lanes_of(bsuite_id)
    for k in states:
      states[k][sl] = s[k]
    actions[sl] = a
    filled[sl] += 1
  assert (filled == 1).all()
  _inject_pair(dev, host, states)
  act = torch.from_numpy(actions)
  gpu, cpu = _outputs(dev, dev.step(act.cuda()), n), _outputs(host, host.step(act), n)
  non_robust = 0
  for bsuite_id, (params, s, a) in per.items():
    sl = dev.lanes_of(bsuite_id)
    env = fr.device_envelope('cartpole_swingup', params, s, a)
    sub = lambda o: {k: (sub(v) if isinstance(v, dict) else np.asarray(v)[sl]) for k, v in o.items()}
    non_robust += _check(f'packed {bsuite_id}', 'cartpole_swingup', env, sub(gpu), sub(cpu))
  print(f'\n[float step] packed cartpole_swingup: {n} lanes, {non_robust} with a non-robust decision')


@pytest.mark.parametrize('family', fr.FAMILIES)
def test_bfloat16_observations(family):
  params, states, actions, _ = _subset(family)
  env = fr.device_envelope(family, params, states, actions)
  n = actions.shape[0]
  dev, host = _make(family, n, 'cuda', obs_dtype='bfloat16'), _make(family, n, 'cpu', obs_dtype='bfloat16')
  _inject_pair(dev, host, states)
  act = torch.from_numpy(actions)
  gpu, cpu = _outputs(dev, dev.step(act.cuda()), n), _outputs(host, host.step(act), n)
  _check(f'{family} bfloat16', family, env, gpu, cpu, obs_dtype='bfloat16')
