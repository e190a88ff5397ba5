"""One step of the float-dynamics families (cartpole, cartpole_swingup, mountain_car) with an error envelope.

`reference_step` evaluates one transition with numpy float64 element-wise ops, vectorised over lanes, in the
reference's operation order as `oracle/bsuite_oracle.py` (`_pole_physics`, `_advance_cartpole[_swingup]`,
`_advance_mountain_car`) and `bsb_families.cuh` (`advance_pole`, `CartpoleT::step`, `MountainCar::step`) restate it.
numpy ufuncs round every operation and never fuse one into the next, so this is the reference's arithmetic; only the
trig values and the square are parameters:

  host twin    sin=np.sin, cos=np.cos, square=HOST_SQUARE: glibc and `pow`, as CPython evaluates them.  The host
               path (device='cpu') must equal it bit for bit.
  device twin  square=DEVICE_SQUARE (the exact product the device computes) and sin / cos taken anywhere in
               [correctly rounded - TRIG_ULPS ulp, correctly rounded + TRIG_ULPS ulp].  `device_envelope` evaluates
               the step for every such trig value and keeps, per lane, the smallest and largest value of every
               output.  A device step whose trig is within TRIG_ULPS ulp and whose other operations are the IEEE
               ones in the reference's order lies inside that envelope; an FMA contraction, a reordered expression or
               a single-precision sin / cos does not.

Outputs that read no trig in this step (the pole's x, theta and t, mountain_car's tick, and the observation entries
made from them) have an envelope of one value: the device must reproduce them bit for bit.  A decision (a comparison
that selects a reward, a step type or a clamp) is robust on a lane when it comes out the same everywhere in the
envelope; where it is not, either outcome is a correct device step.

`build_states` makes the states both test files use: edge states where the dynamics or a decision turn on the last
ulp, lanes that measure the device's trig error directly, and random reachable states from a fixed seed.
`inject_states` / `read_states` move them in and out of an environment through its `state_dict()` blob.
"""

import functools

import mpmath
import numpy as np

from bsuite_b200 import _lib
from bsuite_b200 import experiments

FAMILIES = ('cartpole', 'cartpole_swingup', 'mountain_car')
MID, LAST = 1, 2                 # dm_env step types, as the engine writes them
TWO_PI = 2 * np.pi

# The CUDA Math API's maximum error of double-precision sin, cos and sincos, in ulp (NVIDIA's documented figure,
# not measured here).  glibc's are within 1 ulp.
TRIG_ULPS = 2

_MASS_CART, _MASS_POLE, _LENGTH, _FORCE_MAG, _GRAVITY = 1., 0.1, .5, 10., 9.8    # cartpole.py:106-112

POLE_FIELDS = ('x', 'x_dot', 'theta', 'theta_dot', 't')
STATE_FIELDS = dict(cartpole=POLE_FIELDS, cartpole_swingup=POLE_FIELDS, mountain_car=('pos', 'vel', 'tick'))
# bsuite_info() accumulators, in the order the engine stores them
INFO_FIELDS = dict(cartpole=('raw_return', 'best_episode'),
                   cartpole_swingup=('raw_return', 'total_upright', 'best_episode'),
                   mountain_car=('raw_return',))
# what `device_envelope` holds to one value (state fields and observation columns)
EXACT_STATE = dict(cartpole=('x', 'theta', 't'), cartpole_swingup=('x', 'theta', 't'), mountain_car=('tick',))
EXACT_OBS = dict(cartpole=(0, 5), cartpole_swingup=(0, 5, 6), mountain_car=(2,))
ENVELOPE_STATE = dict(cartpole=('x_dot', 'theta_dot'), cartpole_swingup=('x_dot', 'theta_dot'),
                      mountain_car=('pos', 'vel'))


def HOST_SQUARE(v):
  """`v ** 2` on Python floats: CPython calls libm `pow`, which is not always the correctly rounded square.  (numpy
  turns `array ** 2` into a multiplication, so this goes element by element.)"""
  return np.array([a ** 2 for a in np.asarray(v, np.float64).tolist()], np.float64).reshape(np.shape(v))


def DEVICE_SQUARE(v):
  return v * v


def default_params(family, **overrides):
  """The engine fields of `family` (experiments.<family>(**overrides)), which are the reference's constructor
  arguments."""
  make = dict(cartpole=experiments.cartpole, cartpole_swingup=experiments.cartpole_swingup,
              mountain_car=experiments.mountain_car)[family]
  return dict(make(**overrides).fields)


# ------------------------------------------------------------------ one step
def reference_step(family, params, state, action, sin, cos, square):
  """One transition of every lane of `state` (dict of float64 / int arrays: STATE_FIELDS[family], and optionally the
  accumulators episode_return and INFO_FIELDS[family], zero when absent) under `action` (int array).

  Returns a dict: `state` (the new STATE_FIELDS and episode_return), `info` (the new INFO_FIELDS values), `reward`,
  `step_type` (MID or LAST), `discount`, `obs` (float32 [N, K], the observation row of the new state) and
  `decisions` (name -> bool array, every comparison the step branches on); the poles add `x_acc`."""
  action = np.asarray(action, np.int64)
  if family == 'mountain_car':
    return _mountain_car_step(params, state, action, cos)
  return _pole_step(family == 'cartpole_swingup', params, state, action, sin, cos, square)


def _acc(state, name, n):
  return np.asarray(state[name], np.float64) if name in state else np.zeros(n)


def _pole_step(swingup, params, state, action, sin, cos, square):
  x, x_dot, th, th_dot, t = (np.asarray(state[k], np.float64) for k in POLE_FIELDS)
  n = x.shape[0]
  dt = params['timescale']
  # cartpole.py:37-65
  force = (action - 1).astype(np.float64) * _FORCE_MAG
  c, sn = cos(th), sin(th)
  pl = _MASS_POLE * _LENGTH
  m_total = _MASS_CART + _MASS_POLE
  temp = (force + pl * square(th_dot) * sn) / m_total
  th_acc = (_GRAVITY * sn - c * temp) / (_LENGTH * (4 / 3 - _MASS_POLE * square(c) / m_total))
  x_acc = temp - pl * th_acc * c / m_total
  new = dict(x=x + dt * x_dot, x_dot=x_dot + dt * x_acc, theta=np.remainder(th + dt * th_dot, TWO_PI),
             theta_dot=th_dot + dt * th_acc, t=t + dt)
  c1, s1 = cos(new['theta']), sin(new['theta'])
  x_thr, h, t_max = params['x_threshold'], params['height_threshold'], params['max_time']
  episode_return, raw_return = _acc(state, 'episode_return', n), _acc(state, 'raw_return', n)
  best = _acc(state, 'best_episode', n)
  info = {}
  if not swingup:                                             # cartpole.py:140-153
    decisions = {'cos > height_threshold': c1 > h, '|x| < x_threshold': np.abs(new['x']) < x_thr}
    ok = decisions['cos > height_threshold'] & decisions['|x| < x_threshold']
    reward = np.where(ok, 1., 0.)
    done = (new['t'] > t_max) | ~ok
  else:                                                       # cartpole_swingup.py:104-123
    thd_thr, x_rew = params['theta_dot_threshold'], params['x_reward_threshold']
    decisions = {'cos > height_threshold': c1 > h,
                 '|theta_dot| < theta_dot_threshold': np.abs(new['theta_dot']) < thd_thr,
                 '|x| < x_reward_threshold': np.abs(new['x']) < x_rew, '|x| > x_threshold': np.abs(new['x']) > x_thr}
    upright = (decisions['cos > height_threshold'] & decisions['|theta_dot| < theta_dot_threshold']
               & decisions['|x| < x_reward_threshold'])
    reward = -1. * np.abs(action - 1) * params['move_cost']
    reward = np.where(upright, reward + 1., reward)
    info['total_upright'] = _acc(state, 'total_upright', n) + upright
    done = (new['t'] > t_max) | decisions['|x| > x_threshold']
  new['episode_return'] = episode_return + reward
  info['raw_return'] = raw_return + reward
  info['best_episode'] = np.where(done, np.maximum(new['episode_return'], best), best)
  obs = [new['x'] / x_thr, new['x_dot'] / x_thr, s1, c1, new['theta_dot'], new['t'] / t_max]   # cartpole.py:167-177
  if swingup:                                                 # cartpole_swingup.py:137-150
    obs += [np.where(np.abs(new['x']) < params['x_reward_threshold'], 1., -1.),
            np.where(np.abs(new['theta_dot']) < params['theta_dot_threshold'], 1., -1.)]
  out = _result(new, info, reward, done, obs, decisions)
  out['x_acc'] = x_acc
  return out


def _mountain_car_step(params, state, action, cos):
  pos, vel = np.asarray(state['pos'], np.float64), np.asarray(state['vel'], np.float64)
  tick = np.asarray(state['tick'], np.int64) + 1             # mountain_car.py:73-90
  vel = vel + ((action - 1).astype(np.float64) * 0.001 + cos(3 * pos) * -0.0025)
  decisions = {'vel > 0.07': vel > 0.07, 'vel < -0.07': vel < -0.07}
  vel = np.clip(vel, -0.07, 0.07)
  pos = pos + vel
  decisions.update({'pos > 0.6': pos > 0.6, 'pos < -1.2': pos < -1.2})
  pos = np.clip(pos, -1.2, 0.6)
  at_wall = pos == -1.2
  decisions.update({'pos == -1.2': at_wall, 'vel < 0 at the wall': at_wall & (vel < 0.), 'pos >= 0.5': pos >= .5})
  vel = np.where(at_wall, np.clip(vel, 0., 0.07), vel)
  done = decisions['pos >= 0.5'] | (tick >= params['max_steps'])
  reward = np.full(pos.shape, -1.)
  info = dict(raw_return=_acc(state, 'raw_return', pos.shape[0]) + reward)
  obs = [pos, vel, tick / params['max_steps']]               # mountain_car.py:62-64
  return _result(dict(pos=pos, vel=vel, tick=tick), info, reward, done, obs, decisions)


def _result(new, info, reward, done, obs, decisions):
  return dict(state=new, info=info, reward=reward, step_type=np.where(done, LAST, MID).astype(np.int32),
              discount=np.where(done, 0., 1.).astype(np.float32), obs=np.stack(obs, axis=1).astype(np.float32),
              decisions=decisions)


def host_step(family, params, state, action):
  """The host twin: glibc sin / cos and `pow`, like the reference."""
  return reference_step(family, params, state, action, np.sin, np.cos, HOST_SQUARE)


# ------------------------------------------------------------------ correctly rounded trig
_LD_BITS = np.finfo(np.longdouble).nmant + 1


def correctly_rounded(name, v):
  """`name` ('sin' or 'cos') of every element of `v`, correctly rounded to double.

  mpmath at 40 digits decides every value; where numpy has an extended long double (64-bit significand), its sin /
  cos decide the values that lie clear of a rounding boundary, and only those within 2**-58 (relative) of a midpoint
  between two doubles go to mpmath.  Values are deduplicated by bit pattern, so -0.0 keeps its sign."""
  v = np.asarray(v, np.float64)
  bits, inverse = np.unique(v.reshape(-1).view(np.uint64), return_inverse=True)
  u = bits.view(np.float64)
  out = np.empty_like(u)
  if _LD_BITS >= 64:
    ld = getattr(np, name)(u.astype(np.longdouble))
    d = ld.astype(np.float64)
    below = (d.astype(np.longdouble) + np.nextafter(d, -np.inf).astype(np.longdouble)) / 2
    above = (d.astype(np.longdouble) + np.nextafter(d, np.inf).astype(np.longdouble)) / 2
    margin = np.abs(ld) * np.longdouble(2.) ** -58
    unsure = (np.abs(ld - below) <= margin) | (np.abs(ld - above) <= margin) | ~np.isfinite(d)
    out[:] = d
  else:
    unsure = np.ones(u.shape, bool)
  fn = getattr(mpmath, name)
  with mpmath.workdps(40):
    for i in np.flatnonzero(unsure):
      x = float(u[i])
      out[i] = (x if name == 'sin' else 1.) if x == 0. else float(fn(mpmath.mpf(x)))
  return out[inverse].reshape(v.shape)


def nudge(v, n):
  """`v` moved by `n` ulps (np.nextafter, |n| times)."""
  v = np.asarray(v, np.float64)
  for _ in range(abs(int(n))):
    v = np.nextafter(v, np.inf if n > 0 else -np.inf)
  return v


class _TrigTable:
  """Correctly rounded sin / cos of the arguments one step asks for, computed once per argument array."""

  def __init__(self):
    self._memo = {}

  def __call__(self, name, v):
    v = np.asarray(v, np.float64)
    key = (name, v.tobytes())
    if key not in self._memo:
      self._memo[key] = correctly_rounded(name, v)
    return self._memo[key]


def ulp_offsets(family, k=TRIG_ULPS):
  """The (sin offset, cos offset) pairs the envelope spans: (2k+1)**2 for the poles, 2k+1 for mountain_car."""
  sins = (0,) if family == 'mountain_car' else range(-k, k + 1)
  return [(i, j) for i in sins for j in range(-k, k + 1)]


def offset_step(family, params, state, action, offsets, table=None):
  """The device twin with sin / cos at the given ulp offsets from the correctly rounded values."""
  table = table or _TrigTable()
  i, j = offsets
  return reference_step(family, params, state, action, lambda v: nudge(table('sin', v), i),
                        lambda v: nudge(table('cos', v), j), DEVICE_SQUARE)


def device_envelope(family, params, state, action, k=TRIG_ULPS):
  """Per lane, the smallest and largest value of every output over the device twin's trig values.

  Returns a dict: `lo` / `hi` (dicts of state, info and reward arrays, plus `obs` float32 [N, K]), `robust` (bool
  [N]: every decision comes out the same everywhere in the envelope), `decisions` (name -> bool [N], the robust
  outcome where robust) and `center` (the device twin at the correctly rounded values)."""
  table = _TrigTable()
  runs = [offset_step(family, params, state, action, o, table) for o in ulp_offsets(family, k)]
  center = offset_step(family, params, state, action, (0, 0), table)

  def span(get):
    vals = np.stack([get(r) for r in runs])
    return vals.min(axis=0), vals.max(axis=0)

  lo, hi = {}, {}
  for f in STATE_FIELDS[family] + (() if family == 'mountain_car' else ('episode_return',)):
    lo[f], hi[f] = span(lambda r, f=f: r['state'][f])
  for f in INFO_FIELDS[family]:
    lo['info.' + f], hi['info.' + f] = span(lambda r, f=f: r['info'][f])
  lo['reward'], hi['reward'] = span(lambda r: r['reward'])
  lo['step_type'], hi['step_type'] = span(lambda r: r['step_type'])
  lo['obs'], hi['obs'] = span(lambda r: r['obs'])
  robust = np.ones(np.shape(action), bool)
  for name in center['decisions']:
    d = np.stack([r['decisions'][name] for r in runs])
    robust &= d.all(axis=0) | ~d.any(axis=0)
  return dict(lo=lo, hi=hi, robust=robust, decisions=center['decisions'], center=center)


def outside(env_lo, env_hi, value):
  """True where `value` lies outside [env_lo, env_hi] (NaN counts as outside)."""
  return ~((value >= env_lo) & (value <= env_hi))


# ------------------------------------------------------------------ edge and random states
def _accumulated_times(dt, n):
  """t after 0..n steps of `t += dt`, as the environment accumulates it."""
  out, t = [], 0.
  for _ in range(n + 1):
    out.append(t)
    t += dt
  return np.array(out)


def _pole_states(family, params, n_random, n_trig, rng):
  dt, x_thr, init = params['timescale'], params['x_threshold'], params['init_range']
  thd_thr = params.get('theta_dot_threshold', 1.)
  x_rew = params.get('x_reward_threshold', 1.)
  rows = []                                                   # (x, x_dot, theta, theta_dot, t)
  thetas = [0., -0., 1e-300, -1e-300, 1e-9, -1e-9, init, -init, np.pi / 2, float(nudge(TWO_PI, -1)),
            TWO_PI - 1e-13] + [float(nudge(np.pi, j)) for j in range(-3, 4)]
  theta_dots = [0., 1e-12, -1e-12, 50., -50., 1e3, -1e3] + [
      s * float(nudge(thd_thr, j)) for s in (1., -1.) for j in (-1, 0, 1)]
  rows += [(0., 0., th, thd, 0.) for th in thetas for thd in theta_dots]
  # theta + dt * theta_dot lands on -0.0, on 0.0, just below 0 (the remainder rounds up to 2*pi itself), exactly on
  # 2*pi (the remainder is 0) and a few ulps either side of 2*pi
  small = dt * .1
  rows += [(0., 0., -0., -0., 0.), (0., 0., small, -.1, 0.), (0., 0., float(nudge(small, -1)), -.1, 0.),
           (0., 0., float(nudge(small, 1)), -.1, 0.), (0., 0., 0., -1e-300, 0.), (0., 0., 0., -1e-12, 0.),
           (0., 0., TWO_PI, 0., 0.), (0., 0., TWO_PI - dt, 1., 0.), (0., 0., float(nudge(TWO_PI - dt, 1)), 1., 0.),
           (0., 0., TWO_PI - dt * 3., 3., 0.)]
  # cos(theta') against every height threshold a cartpole or cartpole_swingup setting uses (h = n / 20, 0.8):
  # theta' = +-arccos(h) and 2*pi - arccos(h), +-4 ulps, puts cos(theta') within 16 ulps of h on both sides (within
  # 1 ulp for h >= 0.5)
  for h in sorted({params['height_threshold'], .8} | {n / 20 for n in range(20)}):
    a = float(np.arccos(h))
    for j in range(-4, 5):
      for th in (float(nudge(a, j)), -float(nudge(a, j)), float(nudge(TWO_PI - a, j))):
        rows.append((0., 0., th, 0., 0.))
  # x' on +-x_threshold and +-x_reward_threshold and up to 2 ulps either side, reached with and without a velocity
  for thr in (x_thr, x_rew):
    for s in (1., -1.):
      for j in range(-2, 3):
        rows.append((s * float(nudge(thr, j)), 0., 0., 0., 0.))
        rows.append((s * float(nudge(thr - dt * 1., j)), s * 1., 0., 0., 0.))
  # t one dt before max_time (t' == max_time, not yet past it), and the accumulated times around it
  times = _accumulated_times(dt, int(round(params['max_time'] / dt)) + 2)
  for t in [params['max_time'] - dt] + list(times[-5:]):
    rows.append((0., 0., 0., 0., float(t)))
  edge = np.array(rows, np.float64)
  # trig lanes: theta_dot = 0, x_dot = 0 (with action 1, the new velocities are a function of sin / cos alone)
  trig = np.zeros((n_trig, 5))
  trig[:, 2] = rng.uniform(-init, TWO_PI, n_trig)
  # random reachable states
  r = np.empty((n_random, 5))
  r[:, 0] = rng.uniform(-1.05, 1.05, n_random) * x_thr
  r[:, 1] = rng.standard_normal(n_random) * 2.
  r[:, 2] = rng.uniform(0., TWO_PI, n_random)
  r[:, 2][:n_random // 20] = rng.uniform(-init, init, n_random // 20)      # fresh episodes: theta not yet wrapped
  r[:, 3] = np.where(rng.rand(n_random) < .1, rng.uniform(-60., 60., n_random), rng.standard_normal(n_random) * 3.)
  r[:, 4] = times[rng.randint(0, len(times) - 1, n_random)]
  all_rows = np.concatenate([edge, trig, r])
  states = {f: all_rows[:, k].copy() for k, f in enumerate(POLE_FIELDS)}
  n = all_rows.shape[0]
  states['episode_return'] = rng.randint(0, 1000, n).astype(np.float64)
  states['raw_return'] = states['episode_return'] + rng.randint(0, 1000, n)
  states['best_episode'] = rng.randint(0, 1000, n).astype(np.float64)
  if family == 'cartpole_swingup':
    states['episode_return'] *= .1                # swing-up returns are multiples of 0.1 in practice: not integers
    states['total_upright'] = rng.randint(0, 1000, n).astype(np.float64)
  return states, np.arange(n) - len(edge), len(edge)


def mountain_car_velocity(pos, vel, action):
  """vel' of one mountain_car step before the wall clamp, in the step's own arithmetic (glibc cos)."""
  vel = vel + ((np.asarray(action) - 1).astype(np.float64) * .001 + np.cos(3 * np.asarray(pos)) * -.0025)
  return np.clip(vel, -.07, .07)


def mountain_car_unclamped_position(pos, vel, action):
  """pos + vel' of one mountain_car step: the new position before its clamp to [-1.2, 0.6]."""
  return pos + mountain_car_velocity(pos, vel, action)


def _mountain_car_start_landing_on(target, vel, action):
  """The position p from which `action` at velocity `vel` moves the car to p + vel'(p) == target: the fixed point of
  p <- target - vel'(p) (vel' barely depends on p, so a few iterations converge), then the ulp neighbour that lands
  exactly on `target` where one does."""
  p = target - vel
  for _ in range(20):
    p = float(target - mountain_car_velocity(p, vel, action))
  for j in (0, -1, 1, -2, 2):
    if float(mountain_car_unclamped_position(float(nudge(p, j)), vel, action)) == target:
      return float(nudge(p, j))
  return p


def _mountain_car_states(params, n_random, n_trig, rng):
  max_steps = params['max_steps']
  rows = []                                                   # (pos, vel, tick)
  positions = [-1.2, float(nudge(-1.2, 1)), float(nudge(-1.2, 2)), np.pi / 6, -np.pi / 6, .5, float(nudge(.5, -1)),
               .6, 0.]
  velocities = [0., .07, -.07, 1e-17, -1e-17] + [s * float(nudge(.07, j)) for s in (1., -1.) for j in (-1, 1)]
  rows += [(p, v, 0) for p in positions for v in velocities]
  # The new position (before its clamp) on the goal line 0.5 and on the left wall -1.2, and up to 4 ulps either
  # side: for each action, the position from which that action lands exactly there, then nudged.  Towards the wall
  # the velocity is negative, so these lanes also reach the wall's velocity clamp.
  for target, vels in ((.5, (.01, .03, .0695)), (-1.2, (-.01, -.03, -.0695))):
    for v in vels:
      for a in range(3):
        p = _mountain_car_start_landing_on(target, v, a)
        rows += [(float(nudge(p, j)), v, 0) for j in range(-4, 5)]
  rows += [(p, v, max_steps - 1) for p in (-.5, .49, float(nudge(.5, -1))) for v in (0., .01)]
  edge = np.array(rows, np.float64)
  trig = np.zeros((n_trig, 3))                                # vel = 0: with action 1, vel' = cos(3 pos) * -0.0025
  trig[:, 0] = rng.uniform(-1.2, .6, n_trig)
  r = np.empty((n_random, 3))
  r[:, 0] = rng.uniform(-1.2, .6, n_random)
  r[:, 1] = rng.uniform(-.07, .07, n_random)
  r[:, 2] = rng.randint(0, max_steps, n_random)
  all_rows = np.concatenate([edge, trig, r])
  states = dict(pos=all_rows[:, 0].copy(), vel=all_rows[:, 1].copy(), tick=all_rows[:, 2].astype(np.int64))
  states['raw_return'] = -rng.randint(0, 10 ** 6, all_rows.shape[0]).astype(np.float64)
  return states, np.arange(all_rows.shape[0]) - len(edge), len(edge)


def build_states(family, params, n_random=100_000, n_trig=4096, seed=0):
  """Edge states, trig lanes and `n_random` random reachable states of `family`, each paired with every action.

  Returns (state dict with N = 3 * states lanes, action int32 [N], kind int8 [N]: 0 edge, 1 trig lane, 2 random)."""
  rng = np.random.RandomState(seed)
  if family == 'mountain_car':
    states, index, n_edge = _mountain_car_states(params, n_random, n_trig, rng)
  else:
    states, index, n_edge = _pole_states(family, params, n_random, n_trig, rng)
  kind = np.where(index < 0, 0, np.where(index < n_trig, 1, 2)).astype(np.int8)
  n = kind.shape[0]
  tiled = {k: np.tile(v, 3) for k, v in states.items()}
  return tiled, np.repeat(np.arange(3, dtype=np.int32), n), np.tile(kind, 3)


N_RANDOM = 100_000            # random reachable states per family in the shared case


@functools.lru_cache(maxsize=None)
def cached_case(family):
  """(params, states, actions, kind) of `build_states(family, default_params(family), N_RANDOM)`, built once per
  session: both test files check the same lanes."""
  params = default_params(family)
  states, actions, kind = build_states(family, params, n_random=N_RANDOM)
  return params, states, actions, kind


@functools.lru_cache(maxsize=None)
def cached_envelope(family):
  """`device_envelope` of `cached_case(family)`."""
  params, states, actions, _ = cached_case(family)
  return device_envelope(family, params, states, actions)


def _bits(a):
  a = np.ascontiguousarray(a)
  return a.view({8: np.uint64, 4: np.uint32}[a.dtype.itemsize]) if a.dtype.kind == 'f' else a


def mismatch(got, want):
  """Lanes where `got` and `want` differ bit for bit (rows of 2-D arrays as a whole; -0.0 differs from 0.0)."""
  d = _bits(np.asarray(got)) != _bits(np.asarray(want, dtype=np.asarray(got).dtype))
  return d.reshape(d.shape[0], -1).any(axis=1)


def select(states, lanes):
  """The lanes `lanes` (index or mask) of a state dict."""
  return {k: v[lanes] for k, v in states.items()}


# ------------------------------------------------------------------ the state_dict() blob
def blob_layout(env):
  """Byte offsets of the lane state in `env.state_dict()['blob']`, in the allocation order of `bsb_create`
  (bsb_engine.cu): int64 steps_done, u32 st_word[B], f64 st_f64[F][B] (F = 6 for the poles: x, x_dot, theta,
  theta_dot, t, episode_return; 2 for mountain_car: pos, vel), f64 info[BSB_MAX_INFO][B], then the Logging
  accumulators (track_episodes: 5 columns, 6 on a same-step handle), the RNG stream positions u64[B] and, for
  MT19937, the keys u32[624][B] and indices i32[B].  Asserts that these add up to the blob's size."""
  B = env.batch
  nf = 2 if env.family == _lib.MOUNTAIN_CAR else 6
  word = 8
  f64 = word + 4 * B
  info = f64 + 8 * nf * B
  end = info + 8 * 4 * B
  if env._track:                                              # pylint: disable=protected-access
    end += 8 * (6 if env.autoreset == 'same_step' else 5) * B
  end += 8 * B
  if env._rng_kind == _lib.RNG_MT19937:                       # pylint: disable=protected-access
    end += 4 * 624 * B + 4 * B
  return dict(word=word, f64=f64, nf=nf, info=info, end=end)


def _family_name(env):
  return {_lib.CARTPOLE: 'cartpole', _lib.CARTPOLE_SWINGUP: 'cartpole_swingup', _lib.MOUNTAIN_CAR: 'mountain_car'}[
      env.family]


def inject_states(env, states, lanes=None):
  """A state_dict() of `env` whose lanes `lanes` (default: all) hold `states`, with needs-reset cleared: the next
  step() is a transition from exactly these states.  The other lanes keep what they hold."""
  sd = env.state_dict()
  blob = sd['blob'].copy()
  lay = blob_layout(env)
  assert blob.nbytes == lay['end'], (f'state blob of {blob.nbytes} bytes, the layout implies {lay["end"]}: '
                                     'bsb_create allocates the lane state differently now')
  B = env.batch
  lanes = np.arange(B) if lanes is None else np.arange(B)[lanes]
  family = _family_name(env)
  word = blob[lay['word']:lay['f64']].view(np.uint32).copy()
  f64 = blob[lay['f64']:lay['info']].copy().view(np.float64).reshape(lay['nf'], B)
  info = blob[lay['info']:lay['info'] + 32 * B].copy().view(np.float64).reshape(4, B)
  if family == 'mountain_car':
    word[lanes] = np.asarray(states['tick'], np.uint32) & np.uint32(0x7fffffff)
    f64[0, lanes], f64[1, lanes] = states['pos'], states['vel']
  else:
    word[lanes] = 0
    for k, f in enumerate(POLE_FIELDS):
      f64[k, lanes] = states[f]
    f64[5, lanes] = states.get('episode_return', 0.)
  for k, f in enumerate(INFO_FIELDS[family]):
    info[k, lanes] = states.get(f, 0.)
  blob[lay['word']:lay['f64']] = word.view(np.uint8)
  blob[lay['f64']:lay['info']] = f64.reshape(-1).view(np.uint8)
  blob[lay['info']:lay['info'] + 32 * B] = info.reshape(-1).view(np.uint8)
  return dict(sd, blob=blob)


def read_states(env):
  """The lane state of `env` from its state_dict() blob: STATE_FIELDS, episode_return (poles), INFO_FIELDS and
  `needs_reset`, one array each."""
  blob = env.state_dict()['blob']
  lay = blob_layout(env)
  assert blob.nbytes == lay['end']
  B = env.batch
  family = _family_name(env)
  word = blob[lay['word']:lay['f64']].view(np.uint32).copy()
  f64 = blob[lay['f64']:lay['info']].copy().view(np.float64).reshape(lay['nf'], B)
  info = blob[lay['info']:lay['info'] + 32 * B].copy().view(np.float64).reshape(4, B)
  out = dict(needs_reset=(word >> 31).astype(bool))
  if family == 'mountain_car':
    out.update(pos=f64[0], vel=f64[1], tick=(word & 0x7fffffff).astype(np.int64))
  else:
    out.update({f: f64[k] for k, f in enumerate(POLE_FIELDS)}, episode_return=f64[5])
  out.update({f: info[k] for k, f in enumerate(INFO_FIELDS[family])})
  return out
