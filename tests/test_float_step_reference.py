"""The one-step reference of the float-dynamics families (tests/float_step_reference.py), pinned and given teeth.

* The host path (device='cpu') equals the host twin bit for bit from the edge and random states, for every action:
  step type, reward, discount, observation, the state read back through state_dict() and bsuite_info().  The host
  path is what the golden fixtures pin to the reference, so this ties the helper to the reference's arithmetic.
* The host twin lies inside the device envelope everywhere, and the outputs the envelope calls exact are exact:
  glibc's sin / cos are within TRIG_ULPS ulp of the correctly rounded values on these states.
* The edge states reach the boundaries they are built for: mountain_car's new position lands exactly on the goal
  line 0.5 and on the left wall -1.2 and an ulp either side, the pole's x' on its thresholds, theta' on -0.0 and 2*pi,
  cos(theta') next to every height threshold; so a device that compared with `>` for `>=` or clamped differently
  at the wall would be caught on robust lanes.
* Device twins with the faults a device build could plausibly have (single-precision trig, trig rounded to float32,
  a contracted FMA in the x_dot update) leave the envelope on enough states that tests/test_float_step_gpu.py, which
  holds the CUDA step to the envelope, would catch them.
"""

import fractions

import numpy as np
import pytest
import torch

import bsuite_b200
from tests import float_step_reference as fr

N_MT_RANDOM = 2_001          # MT19937 handles carry 2.5 KB of key per lane: edge states and a slice of the random ones


def _run_host(family, rng, states, actions):
  env = bsuite_b200.make(family, batch=actions.shape[0], device='cpu', seed=5, rng=rng,
                         engine_kwargs=dict(reward_dtype='float64'))
  env.reset()
  env.load_state_dict(fr.inject_states(env, states))
  ts = env.step(torch.from_numpy(actions))
  return env, ts


@pytest.mark.parametrize('rng', ['philox', 'mt19937'])
@pytest.mark.parametrize('family', fr.FAMILIES)
def test_host_path_matches_host_twin_bit_for_bit(family, rng):
  params, states, actions, kind = fr.cached_case(family)
  if rng == 'mt19937':
    # the first N_MT_RANDOM / 3 random states of each action's block
    first = np.zeros_like(kind, bool)
    for a in range(3):
      first[np.flatnonzero((kind == 2) & (actions == a))[:N_MT_RANDOM // 3]] = True
    lanes = (kind < 2) | first
    states, actions = fr.select(states, lanes), actions[lanes]
  env, ts = _run_host(family, rng, states, actions)
  want = fr.host_step(family, params, states, actions)
  got = fr.read_states(env)
  n = actions.shape[0]
  checks = dict(step_type=(ts.step_type.numpy(), want['step_type']), reward=(ts.reward.numpy(), want['reward']),
                discount=(ts.discount.numpy(), want['discount']),
                obs=(ts.observation.numpy().reshape(n, -1), want['obs']))
  checks.update({f: (got[f], want['state'][f]) for f in fr.STATE_FIELDS[family]})
  if family != 'mountain_car':
    checks['episode_return'] = (got['episode_return'], want['state']['episode_return'])
  info = env.bsuite_info()
  checks.update({'info.' + f: (info[f].numpy(), want['info'][f]) for f in fr.INFO_FIELDS[family]})
  assert not got['needs_reset'][want['step_type'] == fr.MID].any()
  for name, (g, w) in checks.items():
    bad = np.flatnonzero(fr.mismatch(g, w))
    assert bad.size == 0, (f'{family} {rng}: {name} differs from the host twin on {bad.size} of {n} lanes, first '
                           f'{bad[0]} (action {actions[bad[0]]}): {g[bad[0]]!r} vs {w[bad[0]]!r}')


@pytest.mark.parametrize('family', fr.FAMILIES)
def test_host_twin_lies_in_the_device_envelope(family):
  params, states, actions, _ = fr.cached_case(family)
  env = fr.cached_envelope(family)
  host = fr.host_step(family, params, states, actions)
  for f in fr.EXACT_STATE[family]:
    assert not fr.mismatch(env['lo'][f], env['hi'][f]).any(), f'{f} is not exact in the envelope'
    assert not fr.mismatch(host['state'][f], env['lo'][f]).any(), f
  for col in fr.EXACT_OBS[family]:
    assert not fr.mismatch(env['lo']['obs'][:, col], env['hi']['obs'][:, col]).any(), f'observation column {col}'
  for f in fr.ENVELOPE_STATE[family]:
    assert not fr.outside(env['lo'][f], env['hi'][f], host['state'][f]).any(), f
  assert not fr.outside(env['lo']['obs'], env['hi']['obs'], host['obs']).any()
  robust = env['robust']
  for name, d in env['decisions'].items():
    assert np.array_equal(host['decisions'][name][robust], d[robust]), name
  for f in ('step_type', 'reward'):
    assert np.array_equal(host[f][robust], env['center'][f][robust]), f
  # the edge states sit on the decisions on purpose; the random ones almost never do
  assert robust.mean() > .999


def test_mountain_car_edge_states_meet_the_goal_line_and_the_wall():
  params, states, actions, kind = fr.cached_case('mountain_car')
  robust = fr.cached_envelope('mountain_car')['robust']
  edge = kind == 0
  landed = fr.mountain_car_unclamped_position(states['pos'], states['vel'], actions)
  for target in (.5, -1.2):
    for j in (-1, 0, 1):
      hits = edge & robust & (landed == fr.nudge(target, j))
      assert hits.sum() >= 3, f'no robust edge lane lands {j} ulp from {target} (pos + vel\' before the clamp)'
  # at the wall the new velocity is negative, so the wall's velocity clamp fires
  at_wall = edge & (landed <= -1.2)
  assert (fr.mountain_car_velocity(states['pos'], states['vel'], actions)[at_wall] < 0).all()


@pytest.mark.parametrize('family', ('cartpole', 'cartpole_swingup'))
def test_pole_edge_states_meet_their_boundaries(family):
  params, states, actions, kind = fr.cached_case(family)
  edge = kind == 0
  dt = params['timescale']
  x1 = states['x'] + dt * states['x_dot']
  for thr in (params['x_threshold'], params.get('x_reward_threshold', 1.)):
    for j in range(-2, 3):
      assert (edge & (np.abs(x1) == fr.nudge(thr, j))).any(), (thr, j)
  raw = states['theta'] + dt * states['theta_dot']
  wrapped = np.remainder(raw, fr.TWO_PI)
  assert (edge & (raw == 0) & np.signbit(raw)).any() and (edge & (raw == 0) & ~np.signbit(raw)).any()
  assert (edge & (raw < 0) & (wrapped == fr.TWO_PI)).any()
  assert (edge & (raw == fr.TWO_PI) & (wrapped == 0)).any()
  near = np.abs(raw - fr.TWO_PI) <= 4 * np.spacing(fr.TWO_PI)
  assert (edge & near & (raw < fr.TWO_PI)).any() and (edge & near & (raw > fr.TWO_PI)).any()
  c1 = np.cos(wrapped)
  for h in [n / 20 for n in range(1, 20)] + [.8]:
    d = (c1 - h)[edge]
    tol = 16 * np.spacing(h) if h < .5 else np.spacing(h)
    assert ((d < 0) & (d >= -tol)).any() and ((d > 0) & (d <= tol)).any(), h


def _leaves(family, run):
  """Lanes where a device-twin run lies outside the envelope (any envelope field, exact field or observation)."""
  env = fr.cached_envelope(family)
  out = np.zeros(run['reward'].shape, bool)
  for f in fr.ENVELOPE_STATE[family] + fr.EXACT_STATE[family]:
    out |= fr.outside(env['lo'][f], env['hi'][f], run['state'][f])
  return out | fr.outside(env['lo']['obs'], env['hi']['obs'], run['obs']).any(axis=1)


def _mutated(family, sin, cos):
  params, states, actions, _ = fr.cached_case(family)
  return fr.reference_step(family, params, states, actions, sin, cos, fr.DEVICE_SQUARE)


@pytest.mark.parametrize('family', fr.FAMILIES)
def test_float32_trig_leaves_the_envelope(family):
  """sin / cos evaluated in float32 (a device that regressed to sincosf / cosf) leaves the envelope on 99.9 % of
  cartpole lanes, 99.9 % of cartpole_swingup lanes and 97.9 % of mountain_car lanes."""
  f32 = lambda fn: (lambda v: fn(np.asarray(v).astype(np.float32)).astype(np.float64))
  frac = _leaves(family, _mutated(family, f32(np.sin), f32(np.cos))).mean()
  assert frac > .95, frac


@pytest.mark.parametrize('family', fr.FAMILIES)
def test_trig_rounded_to_float32_leaves_the_envelope(family):
  """Correct double sin / cos rounded to float32 before use leaves the envelope on 99.8 % of cartpole lanes,
  99.8 % of cartpole_swingup lanes and 97.9 % of mountain_car lanes."""
  r32 = lambda fn: (lambda v: fn(v).astype(np.float32).astype(np.float64))
  frac = _leaves(family, _mutated(family, r32(np.sin), r32(np.cos))).mean()
  assert frac > .95, frac


def _fma(a, b, c):
  """a * b + c rounded once (Python 3.12 has no math.fma)."""
  return float(fractions.Fraction(a) * fractions.Fraction(b) + fractions.Fraction(c))


@pytest.mark.parametrize('family', ('cartpole', 'cartpole_swingup'))
def test_contracted_x_dot_update_leaves_the_envelope(family):
  """x_dot' = x_dot + dt * x_acc computed as one FMA (a unit built without --fmad=false), everything else as the
  device twin at the correctly rounded trig: 3.6 % of the random lanes leave the envelope (10 727 of 300 000, for
  either family)."""
  params, states, actions, kind = fr.cached_case(family)
  env = fr.cached_envelope(family)
  center = env['center']
  lanes = np.flatnonzero(kind == 2)
  dt = params['timescale']
  fused = np.array([_fma(dt, a, v) for a, v in zip(center['x_acc'][lanes].tolist(), states['x_dot'][lanes].tolist())])
  out = fr.outside(env['lo']['x_dot'][lanes], env['hi']['x_dot'][lanes], fused)
  assert out.mean() > .01, out.mean()
