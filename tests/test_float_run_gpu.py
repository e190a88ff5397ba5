"""Whole float-dynamics runs on the device: every step in the one-step envelope, every launch path bit for bit
against single steps, accumulators and log rows exact.

tests/test_float_step_gpu.py pins ONE device step of cartpole, cartpole_swingup and mountain_car to the envelope of
a numpy float64 step (CUDA's sin / cos within 2 ulp).  Longer runs elsewhere are compared with the host path within
FLOAT_TOL, because device and host trig differ in the last ulp and trajectories drift apart.  Here:

  (a) the canonical run: T single step() calls on a CUDA handle from injected edge and random states
      (float_step_reference.build_states).  Before each step the device's blob goes into a device='cpu' twin; after
      it every stepping lane is checked with test_float_step_gpu._check (x, theta, t, tick bit-exact, the rest in the
      envelope, decisions and accumulators exact where robust) and every resetting lane is exact.  So the one-step
      guarantee holds for the states the dynamics reach, over many resets.
  (b) every other launch path (fused rollouts with caller and sampled actions, Philox / MT19937, tracked or not,
      float32 rewards, masked steps, masked rollouts with episode budgets, same-step, packed, bfloat16, CUDA graphs,
      step_host) from the same blob with the same actions: bit for bit equal to the canonical run.  The paths share
      the __host__ __device__ transition and are built with --fmad=false, so nothing may drift between them.
  (c) bsuite_info(), episode_stats() and the log rows equal float_run_reference.expected_accumulators of the run's
      own rewards and step types, bit for bit, over 1 000 episodes per lane, and the device scores the rows as the
      host path does.
"""

import functools

import numpy as np
import pytest
import torch

import bsuite_b200
from bsuite_b200 import analysis
from bsuite_b200 import registry
from bsuite_b200.environment import StepBuffers
from tests import float_run_reference as frr
from tests import float_step_reference as fr
from tests import gauss_draw_reference as gr
from tests import test_float_step_gpu as tfs
from tests import test_scores_gpu as tsg

pytestmark = pytest.mark.gpu

SEED = 11
SHORT = dict(cartpole=dict(max_time=.2), cartpole_swingup=dict(max_time=.2), mountain_car=dict(max_steps=9))
# (batch, calls, episode parameters) of the two canonical runs per family
CASES = dict(short=(4099, 48, SHORT), default=(256, 1100, dict(cartpole={}, cartpole_swingup={}, mountain_car={})))
RUNS = [(f, c) for f in fr.FAMILIES for c in CASES]
RUN_IDS = [f'{f}-{c}' for f, c in RUNS]


def _make(family, batch, device, params, **kw):
  kw = dict(dict(reward_dtype='float64', record_rows=True), **kw)
  rng = kw.pop('rng', 'philox')
  return bsuite_b200.make(family, batch=batch, device=device, seed=SEED, rng=rng, engine_kwargs=kw, **params)


def _start_states(family, params, batch):
  """Edge states, 64 trig lanes and random reachable states of `family`, `batch` of them."""
  states, _, kind = fr.build_states(family, params, n_random=batch, n_trig=64, seed=5)
  n = kind.shape[0] // 3                               # build_states pairs every state with each of 3 actions
  lanes = np.concatenate([np.flatnonzero(kind[:n] == k) for k in (0, 1, 2)])[:batch]
  return fr.select(states, lanes)


# ------------------------------------------------------------------ recording a run
def _part(buf, t, n=None):
  """Rows t (n None: a single-step buffer) or t..t+n of [T, ...] buffers."""
  cut = lambda x: None if x is None else (x[t] if n is None else x[t:t + n])
  return StepBuffers(cut(buf.observation), cut(buf.reward), cut(buf.discount), cut(buf.step_type),
                     None if n is None else cut(buf.actions), cut(buf.final_observation))


def _obs_bits(x):
  x = x.cpu()
  if x.dtype == torch.bfloat16:
    return x.view(torch.int16).numpy().reshape(x.shape[0], x.shape[1], -1)
  return x.numpy().reshape(x.shape[0], x.shape[1], -1)


def _result(env, buf):
  """Every output of a run as numpy arrays, and what it left behind."""
  torch.cuda.synchronize()
  out = dict(obs=_obs_bits(buf.observation), reward=buf.reward.cpu().numpy(), discount=buf.discount.cpu().numpy(),
             step_type=buf.step_type.cpu().numpy(), blob=env.state_dict()['blob'],
             info={k: v.cpu().numpy() for k, v in env.bsuite_info().items()})
  if buf.actions is not None:
    out['actions'] = buf.actions.cpu().numpy()
  if buf.final_observation is not None:
    out['final_obs'] = _obs_bits(buf.final_observation)
  if env._track:                                       # pylint: disable=protected-access
    out['stats'] = {k: v.cpu().numpy() for k, v in env.episode_stats().items()}
  if env._log_schedule is not None:                    # pylint: disable=protected-access
    logged = env.logged_rows()
    out['rows'], out['counts'] = logged['rows'].cpu().numpy(), logged['counts'].cpu().numpy()
  return out


def _differ(label, got, want):
  """Asserts `got` equals `want` bit for bit ([T, B, ...] or [B, ...]); names the first differing step and lane."""
  got, want = np.asarray(got), np.asarray(want)
  assert got.shape == want.shape, f'{label}: shape {got.shape} vs {want.shape}'
  g = np.ascontiguousarray(got)
  w = np.ascontiguousarray(want.astype(got.dtype))
  if g.dtype.kind == 'f':
    bits = {8: np.uint64, 4: np.uint32, 2: np.uint16}[g.dtype.itemsize]
    bad = g.view(bits) != w.view(bits)
  else:
    bad = g != w
  if bad.any():
    where = np.argwhere(bad)[0]
    raise AssertionError(f'{label}: differs at {bad.sum()} entries, first at index {tuple(where)}: '
                         f'{g[tuple(where)]!r} vs {w[tuple(where)]!r}')


def _same_run(label, got, want, keys=('obs', 'reward', 'discount', 'step_type'), end=True):
  for k in keys:
    _differ(f'{label}: {k}', got[k], want[k])
  if not end:
    return
  for k, v in want['info'].items():
    _differ(f'{label}: bsuite_info {k}', got['info'][k], v)
  for k, v in want.get('stats', {}).items():
    if 'stats' in got:
      _differ(f'{label}: episode_stats {k}', got['stats'][k], v)
  if 'rows' in want and 'rows' in got:
    _differ(f'{label}: log rows', got['rows'].transpose(2, 0, 1), want['rows'].transpose(2, 0, 1))
    _differ(f'{label}: row counts', got['counts'], want['counts'])


LANE_SECTIONS = ('st_word', 'st_f64', 'info', 'rng_pos', 'log_next', 'mt_key', 'mt_idx')


def _lane_sections(env, blob):
  sec = gr.blob_sections(env)
  return {k: gr.section(blob, sec, k) for k in LANE_SECTIONS if k in sec}


def _same_blob(label, env, got, want):
  """Blobs bit for bit, except a reward-noise cache whose has-gauss flag is clear: stale by design (a fused rollout
  keeps the lane's stream in registers and may leave a different stale value)."""
  sec = gr.blob_sections(env)
  for name in sec:
    a, b = gr.section(got, sec, name), gr.section(want, sec, name)
    if name == 'wrng_gauss':
      streams = gr.Streams(env, 'wrapper')
      has_a, has_b = streams.read(got)['has'].astype(bool), streams.read(want)['has'].astype(bool)
      _differ(f'{label}: blob has-gauss flags', has_a, has_b)
      a, b = a[has_a], b[has_b]
    _differ(f'{label}: blob {name}', a, b)


def _derived_stats(env, blob):
  """The five Logging columns held in `blob` (bsb_families.cuh:661-670)."""
  sec = gr.blob_sections(env)
  ep, calls = gr.section(blob, sec, 'ep'), float(gr.section(blob, sec, 'steps_done'))
  return dict(steps=calls - ep[3], episode=ep[1], total_return=ep[0],
              episode_len=np.where(ep[3] == 0., 0., (calls - 1.) - ep[4]), episode_return=ep[2])


# ------------------------------------------------------------------ (a) the canonical run
def _ulp_offsets(family, params, pre, action, post):
  """Per lane, the smallest max(|sin offset|, |cos offset|) <= TRIG_ULPS that reproduces the device's new velocities
  (TRIG_ULPS + 1 where none does)."""
  fields = ('vel',) if family == 'mountain_car' else ('x_dot', 'theta_dot')
  best = np.full(action.shape[0], fr.TRIG_ULPS + 1)
  table = fr._TrigTable()                              # pylint: disable=protected-access
  for o in fr.ulp_offsets(family):
    run = fr.offset_step(family, params, pre, action, o, table)
    hit = np.all([~fr.mismatch(run['state'][f], post[f]) for f in fields], axis=0)
    best = np.where(hit, np.minimum(best, max(abs(o[0]), abs(o[1]))), best)
  return best


@functools.lru_cache(maxsize=None)
def canonical(family, case):
  """The canonical run of `family` / `case`, checked step by step as (a) of the module docstring.  Returns the
  handle's configuration, its starting state_dict, the actions, the run's outputs (_result), the lane sections and
  derived Logging columns before every call, and the counts the test prints."""
  batch, T, params = CASES[case][0], CASES[case][1], CASES[case][2][family]
  eparams = fr.default_params(family, **params)
  dev, host = _make(family, batch, 'cuda', params), _make(family, batch, 'cpu', params)
  dev.reset()
  sd0 = frr.inject(dev, _start_states(family, eparams, batch))
  dev.load_state_dict(sd0)
  actions = np.random.RandomState(3).randint(0, 3, (T, batch)).astype(np.int32)
  act_dev = torch.from_numpy(actions).cuda()
  buf = dev.make_buffers(T, with_actions=True)
  hbuf = host.make_buffers()
  snaps, stats, blob = [], [], sd0['blob']
  non_robust = lane_steps = resets = 0
  worst = np.zeros(0, int)
  for t in range(T):
    snaps.append(_lane_sections(dev, blob))
    stats.append(_derived_stats(dev, blob))
    host.load_state_dict(dict(sd0, blob=blob))
    pre = frr.lane_state(dev, blob)
    dev.step(act_dev[t], out=_part(buf, t))
    host.step(torch.from_numpy(actions[t]), out=hbuf)
    blob = dev.state_dict()['blob']
    post, hpost = frr.lane_state(dev, blob), frr.lane_state(host, host.state_dict()['blob'])
    gpu = dict(step_type=buf.step_type[t].cpu().numpy(), discount=buf.discount[t].cpu().numpy(),
               reward=buf.reward[t].cpu().numpy(), obs=buf.observation[t].cpu().numpy().reshape(batch, -1),
               state=post, info={f: post[f] for f in fr.INFO_FIELDS[family]})
    cpu = dict(step_type=hbuf.step_type.numpy().copy(), discount=hbuf.discount.numpy().copy(),
               reward=hbuf.reward.numpy().copy(), obs=hbuf.observation.numpy().reshape(batch, -1).copy(),
               state=hpost, info={f: hpost[f] for f in fr.INFO_FIELDS[family]})
    stepping = np.flatnonzero(~pre['needs_reset'])
    if stepping.size:
      st, a = fr.select(pre, stepping), actions[t][stepping]
      env = fr.device_envelope(family, eparams, st, a)
      sub = lambda o: {k: (sub(v) if isinstance(v, dict) else np.asarray(v)[stepping]) for k, v in o.items()}
      non_robust += tfs._check(f'{family} {case} step {t}', family, env, sub(gpu), sub(cpu))   # pylint: disable=protected-access
      worst = np.concatenate([worst, _ulp_offsets(family, eparams, st, a, fr.select(post, stepping))])
      lane_steps += stepping.size
    reset = np.flatnonzero(pre['needs_reset'])
    if reset.size:
      resets += reset.size
      for f in fr.STATE_FIELDS[family] + fr.INFO_FIELDS[family]:
        _differ(f'{family} {case} step {t}: reset {f}', post[f][reset], hpost[f][reset])
      for f in ('step_type', 'discount', 'reward'):
        _differ(f'{family} {case} step {t}: reset {f}', gpu[f][reset], cpu[f][reset])
      lo, hi = tfs._reset_obs_envelope(family, eparams, fr.select(hpost, reset))   # pylint: disable=protected-access
      bad = fr.outside(lo, hi, gpu['obs'][reset]).any(axis=1)
      assert not bad.any(), f'{family} {case} step {t}: reset observation outside its envelope, lane {reset[bad][0]}'
  snaps.append(_lane_sections(dev, blob))
  stats.append(_derived_stats(dev, blob))
  buf.actions.copy_(act_dev)
  res = _result(dev, buf)
  counts = dict(lane_steps=lane_steps, resets=resets, non_robust=non_robust,
                ulp_hist=np.bincount(worst, minlength=fr.TRIG_ULPS + 2))
  return dict(params=params, eparams=eparams, batch=batch, T=T, sd0=sd0, actions=actions, res=res, snaps=snaps,
              stats=stats, counts=counts)


@pytest.mark.parametrize('family,case', RUNS, ids=RUN_IDS)
def test_canonical_run_stays_in_the_envelope(family, case):
  c = canonical(family, case)
  n = c['counts']
  hist = n['ulp_hist']
  print(f'\n[float run] {family} {case}: B={c["batch"]} T={c["T"]}: {n["lane_steps"]} lane-steps in the envelope, '
        f'{n["resets"]} resets exact, {n["non_robust"]} lane-steps with a non-robust decision; largest trig offset '
        f'that reproduces the device step: {dict(enumerate(hist.tolist()))} (>{fr.TRIG_ULPS}: none within the model)')
  episodes = (c['res']['step_type'] == frr.LAST).sum(axis=0)
  assert episodes.min() >= (2 if case == 'short' else 1)


# ------------------------------------------------------------------ (b) every other path, bit for bit
def _fresh(c, family, **kw):
  env = _make(family, c['batch'], 'cuda', c['params'], **kw)
  return env


def _run_segments(env, actions, segments, final=False):
  """A run through `segments` [(kind, length)] with caller actions; returns _result."""
  T = actions.shape[0]
  buf = env.make_buffers(T, with_actions=True, final_observation=final)
  act = torch.from_numpy(actions).cuda()
  t = 0
  for kind, n in segments:
    if kind == 'rollout':
      env.rollout(n, actions=act[t:t + n], out=_part(buf, t, n))
    else:
      for k in range(n):
        env.step(act[t + k], out=_part(buf, t + k))
    t += n
  assert t == T
  buf.actions.copy_(act)
  return _result(env, buf)


@pytest.mark.parametrize('family,case', RUNS, ids=RUN_IDS)
def test_fused_rollouts_equal_single_steps(family, case):
  c = canonical(family, case)
  T = c['T']
  script = frr.run_script(T, c['batch'], 3, seed=1)
  plans = dict(whole=[('rollout', T)], two=[('rollout', 2), ('step', T - 2)],
               thirty_seven=[('rollout', 37), ('rollout', T - 37)],
               mixed=[(k, n) for k, n, _ in script['segments']])
  for name, segments in plans.items():
    env = _fresh(c, family)
    env.load_state_dict(c['sd0'])
    got = _run_segments(env, c['actions'], segments)
    _same_run(f'{family} {case} rollout {name}', got, c['res'])
    _differ(f'{family} {case} rollout {name}: blob', got['blob'], c['res']['blob'])


@pytest.mark.parametrize('family', fr.FAMILIES)
def test_sampled_actions_equal_single_steps(family):
  c = canonical(family, 'short')
  T = c['T']
  a, b = _fresh(c, family), _fresh(c, family)
  a.load_state_dict(c['sd0'])
  b.load_state_dict(c['sd0'])
  buf = a.make_buffers(T, with_actions=True)
  a.rollout(T, action_seed=9, out=buf)
  sampled = _result(a, buf)
  assert np.array_equal(sampled['actions'], b.random_actions(T, action_seed=9))
  got = _run_segments(b, sampled['actions'], [('step', T)])
  _same_run(f'{family} sampled', got, sampled, keys=('obs', 'reward', 'discount', 'step_type', 'actions'))
  _differ(f'{family} sampled: blob', got['blob'], sampled['blob'])


VARIANTS = [('philox', False, 'float64'), ('philox', True, 'float32'), ('mt19937', True, 'float64'),
            ('mt19937', False, 'float32')]


@pytest.mark.parametrize('rng,track,reward_dtype', VARIANTS, ids=['-'.join(map(str, v)) for v in VARIANTS])
@pytest.mark.parametrize('family', fr.FAMILIES)
def test_rng_tracking_and_reward_dtype(family, rng, track, reward_dtype):
  """Single steps against a fused rollout, and against a float64 twin of the same configuration; Philox variants also
  against the canonical run (their blob is the canonical one, less what the variant does not keep)."""
  c = canonical(family, 'short')
  kw = dict(rng=rng, track_episodes=track, record_rows=track, reward_dtype=reward_dtype)
  envs = [_fresh(c, family, **kw) for _ in range(2)] + [_fresh(c, family, **dict(kw, reward_dtype='float64'))]
  if rng == 'philox':
    sds = [frr.transplant(_fresh(c, family), c['sd0']['blob'], e) for e in envs]
  else:
    envs[0].reset()
    sd = frr.inject(envs[0], _start_states(family, c['eparams'], c['batch']))
    sds = [dict(sd)] * 3
  for e, sd in zip(envs, sds):
    e.load_state_dict(sd)
  steps = _run_segments(envs[0], c['actions'], [('step', c['T'])])
  fused = _run_segments(envs[1], c['actions'], [('rollout', c['T'])])
  twin = _run_segments(envs[2], c['actions'], [('step', c['T'])])
  label = f'{family} {rng} track={track} {reward_dtype}'
  _same_run(f'{label} fused', fused, steps)
  _differ(f'{label} fused: blob', fused['blob'], steps['blob'])
  _same_run(f'{label} vs float64 twin', steps, dict(twin, reward=twin['reward'].astype(steps['reward'].dtype)))
  _differ(f'{label} vs float64 twin: blob', steps['blob'], twin['blob'])
  if rng == 'philox':
    want = dict(c['res'], reward=c['res']['reward'].astype(steps['reward'].dtype))
    _same_run(f'{label} vs canonical', steps, want)


@pytest.mark.parametrize('family', fr.FAMILIES)
def test_masked_steps(family):
  """A changing mask: lane i's k-th active call is the canonical run's call k of lane i; lanes that sit out keep
  every byte of their state (the Logging counters move by design: their derived columns do not)."""
  c = canonical(family, 'short')
  B, T, res = c['batch'], c['T'], c['res']
  env = _fresh(c, family)
  env.load_state_dict(c['sd0'])
  k = np.zeros(B, np.int64)
  rng = np.random.RandomState(8)
  out = env.make_buffers()
  lanes = np.arange(B)
  for call in range(2 * T):
    mask = (rng.rand(B) < (.5, .9, .1, 1.)[call % 4]) & (k < T)
    a = c['actions'][np.minimum(k, T - 1), lanes]
    before = env.state_dict()['blob']
    before_stats = _derived_stats(env, before)
    env.step(torch.from_numpy(a).cuda(), out=out, mask=torch.from_numpy(mask).cuda())
    torch.cuda.synchronize()
    on = np.flatnonzero(mask)
    for name, got in (('obs', out.observation.cpu().numpy().reshape(B, -1)), ('reward', out.reward.cpu().numpy()),
                      ('discount', out.discount.cpu().numpy()), ('step_type', out.step_type.cpu().numpy())):
      _differ(f'{family} masked call {call}: {name}', got[on], res[name][k[on], on])
    after = env.state_dict()['blob']
    off = np.flatnonzero(~mask)
    sa, sb = _lane_sections(env, after), _lane_sections(env, before)
    for name in sa:
      _differ(f'{family} masked call {call}: sat-out lanes changed {name}', sa[name][..., off], sb[name][..., off])
    da = _derived_stats(env, after)
    for name in da:
      _differ(f'{family} masked call {call}: sat-out lanes changed {name}', da[name][off], before_stats[name][off])
    k[on] += 1
  final = _lane_sections(env, env.state_dict()['blob'])
  for name, v in final.items():
    want = np.stack([c['snaps'][int(k[i])][name][..., i] for i in range(B)], axis=-1)
    _differ(f'{family} masked: final {name}', v, want)
  stats = {n: v.cpu().numpy() for n, v in env.episode_stats().items()}
  for name, v in stats.items():
    _differ(f'{family} masked: final {name}', v, np.array([c['stats'][int(k[i])][name][i] for i in range(B)]))


SENTINEL = dict(obs=-5., reward=-123., discount=-1., step_type=7)


@pytest.mark.parametrize('family', fr.FAMILIES)
def test_masked_rollouts_with_episode_budgets(family):
  c = canonical(family, 'short')
  B, T, res = c['batch'], c['T'], c['res']
  script = frr.run_script(T, B, 3, seed=6, segments=(7, 11, 5), masks=True, budgets=True)
  env = _fresh(c, family)
  env.load_state_dict(c['sd0'])
  left = script['budgets'].copy()
  left_dev = torch.from_numpy(left.copy()).cuda()
  k = np.zeros(B, np.int64)
  lanes = np.arange(B)
  last = res['step_type'] == frr.LAST
  for j, (_, n, mask) in enumerate(script['segments']):
    idx = np.minimum(k[None] + np.arange(n)[:, None], T - 1)
    acts = c['actions'][idx, lanes]
    out = env.make_buffers(n, with_actions=True)
    for name, v in (('observation', 'obs'), ('reward', 'reward'), ('discount', 'discount'), ('step_type', 'step_type')):
      getattr(out, name).fill_(SENTINEL[v])
    env.rollout(n, actions=torch.from_numpy(acts).cuda(), out=out, mask=torch.from_numpy(mask).cuda(),
                episodes_left=left_dev)
    torch.cuda.synchronize()
    # the active steps of lane i: a prefix, up to the LAST that spends its budget
    active = np.zeros((n, B), bool)
    for i in np.flatnonzero(mask & (left > 0)):
      ends = np.flatnonzero(last[k[i]:k[i] + n, i])
      m = n if ends.size < left[i] else ends[left[i] - 1] + 1
      active[:m, i] = True
    used = active.sum(axis=0)
    spent = np.array([last[k[i]:k[i] + used[i], i].sum() for i in range(B)])
    got = dict(obs=out.observation.cpu().numpy().reshape(n, B, -1), reward=out.reward.cpu().numpy(),
               discount=out.discount.cpu().numpy(), step_type=out.step_type.cpu().numpy())
    for name, g in got.items():
      want = res[name][idx, lanes]
      want = np.where(active.reshape(active.shape + (1,) * (want.ndim - 2)), want, SENTINEL[name])
      _differ(f'{family} masked rollout launch {j}: {name}', g, want.astype(g.dtype))
    left -= spent
    _differ(f'{family} masked rollout launch {j}: episodes_left', left_dev.cpu().numpy(), left)
    k += used
  final = _lane_sections(env, env.state_dict()['blob'])
  for name, v in final.items():
    want = np.stack([c['snaps'][int(k[i])][name][..., i] for i in range(B)], axis=-1)
    _differ(f'{family} masked rollout: final {name}', v, want)
  stats = {n: v.cpu().numpy() for n, v in env.episode_stats().items()}
  for name, v in stats.items():
    _differ(f'{family} masked rollout: final {name}', v, np.array([c['stats'][int(k[i])][name][i] for i in range(B)]))


@pytest.mark.parametrize('fused', [False, True], ids=['steps', 'fused'])
@pytest.mark.parametrize('family', fr.FAMILIES)
def test_same_step_handle_is_the_folded_canonical_run(family, fused):
  """The call after each LAST is dropped; the LAST returns the next FIRST's observation and its own as
  final_observation."""
  c = canonical(family, 'short')
  B, T, res = c['batch'], c['T'], c['res']
  st = res['step_type']
  maps = []
  for i in range(B):
    m, t = [], 0
    while t < T and (st[t, i] != frr.LAST or t + 1 < T):
      m.append(t)
      t += 2 if st[t, i] == frr.LAST else 1
    maps.append(m)
  J = min(len(m) for m in maps)
  idx = np.array([m[:J] for m in maps]).T                 # [J, B] canonical call of each same-step call
  lanes = np.arange(B)
  env = _fresh(c, family, autoreset='same_step', track_episodes=False, record_rows=False)
  env.load_state_dict(frr.transplant(_fresh(c, family), c['sd0']['blob'], env))
  got = _run_segments(env, c['actions'][idx, lanes], [('rollout' if fused else 'step', J)], final=True)
  is_last = st[idx, lanes] == frr.LAST
  for name in ('reward', 'discount', 'step_type'):
    _differ(f'{family} same_step: {name}', got[name], res[name][idx, lanes])
  _differ(f'{family} same_step: obs', got['obs'], res['obs'][np.where(is_last, idx + 1, idx), lanes])
  _differ(f'{family} same_step: final_observation', got['final_obs'][is_last], res['obs'][idx, lanes][is_last])
  end = idx[-1] + np.where(is_last[-1], 2, 1)
  final = _lane_sections(env, got['blob'])
  for name in ('st_word', 'st_f64', 'info', 'rng_pos'):
    want = np.stack([c['snaps'][int(end[i])][name][..., i] for i in range(B)], axis=-1)
    _differ(f'{family} same_step: final {name}', final[name], want)


PACKS = ['cartpole', 'cartpole_swingup', 'mountain_car', 'cartpole_noise', 'cartpole_scale', 'mountain_car_noise',
         'mountain_car_scale']


@pytest.mark.parametrize('experiment', PACKS)
def test_packed_experiment(experiment):
  """Each setting's lanes of the pack (single steps and a fused rollout) against a single-id handle of that setting,
  and the pack's accumulators and rows against expected_accumulators (wrapper-free twin for the unwrapped reward)."""
  L, T = 64, 300
  kw = dict(reward_dtype='float64', record_rows=True)
  pack = registry.load_experiment(experiment, L, device='cuda', seed=SEED, **kw)
  fused = registry.load_experiment(experiment, L, device='cuda', seed=SEED, **kw)
  twin = gr.noise_free_twin(pack)
  family = frr.family_name(pack)
  B = pack.batch
  actions = np.random.RandomState(2).randint(0, 3, (T, B)).astype(np.int32)
  init = frr.initial_state(pack, pack.state_dict()['blob'])
  got = _run_segments(pack, actions, [('step', T)])
  got_fused = _run_segments(fused, actions, [('rollout', 100), ('step', 1), ('rollout', T - 101)])
  _same_run(f'{experiment} pack fused', got_fused, got)
  _same_blob(f'{experiment} pack fused', fused, got_fused['blob'], got['blob'])
  unwrapped = _run_segments(twin, actions, [('step', T)])['reward']
  for k, bsuite_id in enumerate(pack.bsuite_ids):
    sl = pack.lanes_of(bsuite_id)
    single = registry.load_from_id(bsuite_id, batch=L, device='cuda', seed=pack.setting_seeds[k], **kw)
    want = _run_segments(single, actions[:, sl], [('step', T)])
    part = dict(obs=got['obs'][:, sl], reward=got['reward'][:, sl], discount=got['discount'][:, sl],
                step_type=got['step_type'][:, sl], info={n: v[sl] for n, v in got['info'].items()},
                stats={n: v[sl] for n, v in got['stats'].items()}, rows=got['rows'][..., sl],
                counts=got['counts'][sl])
    _same_run(f'{experiment} {bsuite_id}', part, want)
  acc = frr.expected_accumulators(family, got['reward'], got['step_type'], unwrapped, initial=init,
                                  info_names=pack.info_names, log_schedule=pack.logged_rows()['schedule'])
  _same_run(f'{experiment} expected_accumulators', got,
            dict(info=acc.bsuite_info(), stats=acc.episode_stats(), **acc.logged_rows()), keys=())


@pytest.mark.parametrize('family', fr.FAMILIES)
def test_bfloat16_handle(family):
  c = canonical(family, 'short')
  env = _fresh(c, family, obs_dtype='bfloat16')
  env.load_state_dict(c['sd0'])
  got = _run_segments(env, c['actions'], [('step', 5), ('rollout', c['T'] - 5)])
  want = torch.from_numpy(np.ascontiguousarray(c['res']['obs'])).to(torch.bfloat16).view(torch.int16).numpy()
  _same_run(f'{family} bfloat16', got, dict(c['res'], obs=want))
  _differ(f'{family} bfloat16: blob', got['blob'], c['res']['blob'])


@pytest.mark.parametrize('family', fr.FAMILIES)
def test_graph_replay_and_step_host(family):
  c = canonical(family, 'short')
  n = 16
  res = c['res']
  head = lambda name: res[name][:n]
  for fused in (False, True):
    env = _fresh(c, family)
    graphed = env.capture(n, fused=fused)
    env.load_state_dict(c['sd0'])
    graphed.actions.copy_(torch.from_numpy(c['actions'][:n]).cuda())
    ts = graphed.replay()
    torch.cuda.synchronize()
    got = dict(obs=_obs_bits(ts.observation), reward=ts.reward.cpu().numpy(), discount=ts.discount.cpu().numpy(),
               step_type=ts.step_type.cpu().numpy())
    for name in got:
      _differ(f'{family} graph fused={fused}: {name}', got[name], head(name))
    _differ(f'{family} graph fused={fused}: state', _lane_sections(env, env.state_dict()['blob'])['st_f64'],
            c['snaps'][n]['st_f64'])
  env = _fresh(c, family)
  env.load_state_dict(c['sd0'])
  hb = env.make_host_buffers()
  for t in range(n):
    _, obs = env.step_host(torch.from_numpy(c['actions'][t].copy()), hb)
    torch.cuda.synchronize()
    for name, g in (('reward', hb.reward.numpy()), ('discount', hb.discount.numpy()),
                    ('step_type', hb.step_type.numpy()), ('obs', _obs_bits(obs[None])[0])):
      _differ(f'{family} step_host call {t}: {name}', g, res[name][t])
  _differ(f'{family} step_host: state', _lane_sections(env, env.state_dict()['blob'])['st_f64'], c['snaps'][n]['st_f64'])


# ------------------------------------------------------------------ (c) accumulators and rows exact
@pytest.mark.parametrize('family,case', RUNS, ids=RUN_IDS)
def test_canonical_accumulators_are_exact(family, case):
  c = canonical(family, case)
  env = _fresh(c, family)
  res = c['res']
  acc = frr.expected_accumulators(family, res['reward'], res['step_type'], initial=frr.initial_state(env, c['sd0']['blob']),
                                  info_names=env.info_names, log_schedule=env.logged_rows()['schedule'])
  _same_run(f'{family} {case} accumulators', res, dict(info=acc.bsuite_info(), stats=acc.episode_stats(),
                                                       **acc.logged_rows()), keys=())


@pytest.mark.parametrize('family', fr.FAMILIES)
def test_a_thousand_episodes_per_lane(family):
  """Fused rollouts (bit for bit the canonical path, above) from the short case's start until every lane has
  finished 1 000 episodes; the accumulators and all log rows are the model's."""
  c = canonical(family, 'short')
  env = _fresh(c, family)
  env.load_state_dict(c['sd0'])
  acc = frr.Accumulators(family, c['batch'], env.info_names, env.logged_rows()['schedule'],
                         frr.initial_state(env, c['sd0']['blob']))
  chunk = 2000
  buf = env.make_buffers(chunk, with_actions=True)
  launches = 0
  while acc.stats['episode'].min() < 1000:
    env.rollout(chunk, action_seed=launches, out=buf)
    acc.feed(buf.reward.cpu().numpy(), buf.step_type.cpu().numpy())
    launches += 1
    assert launches < 20
  logged = env.logged_rows()
  assert logged['counts'].min().item() == len(logged['schedule'])
  res = _result(env, env.make_buffers(1, with_actions=True))
  _same_run(f'{family} 1000 episodes', res, dict(info=acc.bsuite_info(), stats=acc.episode_stats(),
                                                 **acc.logged_rows()), keys=())
  print(f'\n[float run] {family}: {launches * chunk} calls, {int(acc.stats["episode"].min())}+ episodes per lane, '
        f'rows exact')


@pytest.mark.parametrize('experiment', ['cartpole_noise', 'cartpole_scale'])
def test_scores_of_exact_rows(experiment):
  """A complete run of every setting (1 000 episodes per lane, fused rollouts) on the device: rows equal the model's
  (Logging columns on the wrapped reward, environment columns on the wrapper-free twin's), and the device scores
  them as the host path scores host copies, bit for bit."""
  L = 16
  kw = dict(reward_dtype='float64', record_rows=True)         # ~90 000 calls: up to 100 steps per episode
  env = registry.load_experiment(experiment, L, device='cuda', seed=SEED, **kw)
  twin = gr.noise_free_twin(env)
  family = frr.family_name(env)
  acc = frr.Accumulators(family, env.batch, env.info_names, env.logged_rows()['schedule'],
                         frr.initial_state(env, env.state_dict()['blob']))
  chunk = 10000
  buf, tbuf = env.make_buffers(chunk), twin.make_buffers(chunk)
  launches = 0
  while acc.stats['episode'].min() < 1000:
    actions = torch.from_numpy(np.random.RandomState(launches).randint(0, 3, (chunk, env.batch)).astype(np.int32)).cuda()
    env.rollout(chunk, actions=actions, out=buf)
    twin.rollout(chunk, actions=actions, out=tbuf)
    acc.feed(buf.reward.cpu().numpy(), buf.step_type.cpu().numpy(), tbuf.reward.cpu().numpy())
    launches += 1
    assert launches < 30
  res = _result(env, env.make_buffers(1, with_actions=True))
  _same_run(f'{experiment} rows', res, dict(info=acc.bsuite_info(), stats=acc.episode_stats(), **acc.logged_rows()),
            keys=())
  result = analysis.bsuite_score(env)
  tsg.assert_bitwise(result, analysis.score_rows(tsg.host_copies([(None, env)])))
  assert not torch.isnan(result.score[analysis.EXPERIMENTS.index(experiment)]).any()
