"""Every integer, Bernoulli and uniform draw of a CUDA call against numpy, from injected stream states, on every
launch path that draws (tests/draw_reference.py).

Per call, new stream states go into the handle's blob and into one oracle lane per engine lane; the lane state
carries over.  The device must equal the oracle bit for bit on step type, reward, discount, observation (final
observation where a same-step handle keeps it), the stream word or MT19937 key and index after the call, and
bsuite_info().  Stochastic deep_sea's corner reward passes through randn and is held to noise_reward_tolerance (its
stream word stays exact); the float families are checked at their resets only (observation and drawn state).
"""

import collections
import time

import numpy as np
import pytest
import torch

import bsuite_b200
from bsuite_b200 import datasets
from tests import draw_reference as dr

pytestmark = pytest.mark.gpu

B = 4099                       # 128 full 32-lane chunks and a 3-lane tail
EDGE_COUNTS = collections.Counter()
T0 = time.time()


@pytest.fixture(scope='module')
def mnist_70000(tmp_path_factory):
  path = str(tmp_path_factory.mktemp('draw_mnist_gpu'))
  datasets.write_synthetic_mnist(path, dr.MNIST_IMAGES, 1, seed=3)
  return path


@pytest.fixture(scope='module', autouse=True)
def _report():
  yield
  print(f'\n[draws gpu] lanes per edge class and path: {dict(sorted(EDGE_COUNTS.items()))}')
  print(f'[draws gpu] module time {time.time() - T0:.1f} s')


def _count(path, run):
  for cls, c in run.reached.items():
    EDGE_COUNTS[f'{path}:{cls}'] += c


# ------------------------------------------------------------------ single steps
SINGLE = ([('catch', B, rng, track) for rng in ('philox', 'mt19937') for track in (False, True)]
          + [(n, 1024, rng, track) for n in ('memory_b33', 'umbrella_d65') for rng in ('philox', 'mt19937')
             for track in (False, True)]
          + [(n, 256, rng, False) for n in ('umbrella_d129', 'memory_b64', 'mnist_65537', 'deep_sea_stochastic',
                                            'cartpole', 'mountain_car') for rng in ('philox', 'mt19937')])


@pytest.mark.parametrize('name,batch,rng,track', SINGLE, ids=[f'{n}-{b}-{g}-{"tracked" if t else "untracked"}'
                                                             for n, b, g, t in SINGLE])
def test_single_steps(name, batch, rng, track, mnist_70000):
  """catch at B = 4099 (128 full 32-lane chunks and a 3-lane tail), Philox and MT19937, tracked and not; the other
  configurations at smaller batches: the per-lane Python oracle, not the device, sets the module's run time."""
  run = dr.run_calls(name, rng, 'cuda', mnist_70000, per_class=8, batch=batch, track_episodes=track)
  _count(f'single-{rng}', run)


# ------------------------------------------------------------------ rollouts
def _fresh(name, batch, rng='philox', per_class=8, **kw):
  env = dr.make(name, batch, 'cuda', rng=rng, **kw)
  classes = dr.reachable(env._spec, rng == 'mt19937')               # pylint: disable=protected-access
  r = np.random.RandomState(5)
  return dr.DrawRun(env, dr.lane_plan(classes, per_class, batch, r), seed=5), r


def _reset_all(run):
  run.inject(dr.reset_call)
  ts = run.env.reset()
  dr.check_call(run, 'reset', ts, dr.reset_call, device=True)


def _all_reached(label, run):
  assert not run.unreached().size, f'{label}: lanes {run.unreached()} never reached their class'


@pytest.mark.parametrize('sampled', [False, True], ids=['caller_actions', 'device_actions'])
@pytest.mark.parametrize('rng', ['philox', 'mt19937'])
@pytest.mark.parametrize('name', ['catch_c9', 'umbrella_d9', 'memory_b33'])
def test_rollout(name, rng, sampled):
  """rollout(6) keeps the streams in registers over its steps; MT19937 lanes aim at a regeneration inside a middle
  step (class mt_mid_step)."""
  run = dr.run_rollout(name, rng, 'cuda', sampled, per_class=8, batch=512)
  _count(f'rollout-{"sampled" if sampled else "caller"}-{rng}', run)


# ------------------------------------------------------------------ masked calls
@pytest.mark.parametrize('rng', ['philox', 'mt19937'])
@pytest.mark.parametrize('name', ['catch', 'umbrella_d65'])
def test_masked_step_and_reset(name, rng):
  run, r = _fresh(name, 512, rng)
  _reset_all(run)
  env = run.env
  masks = r.rand(4, env.batch) < 0.6
  run.aim_only(np.flatnonzero(masks[2]))   # every lane of the masked reset draws; a masked step may draw nothing
  for k in range(4):
    mask = masks[k]
    lanes = np.flatnonzero(mask)
    out = env.make_buffers()
    m = torch.from_numpy(mask).cuda()
    if k == 2:
      run.inject(dr.reset_call, lanes)
      ts = env.reset(out=out, mask=m)
      dr.check_call(run, f'{name} {rng} masked reset', ts, dr.reset_call, lanes, device=True)
    else:
      a = r.randint(0, env.num_actions, env.batch).astype(np.int32)
      call = dr.step_call(a)
      run.inject(call, lanes)
      ts = env.step(torch.from_numpy(a).cuda(), out=out, mask=m)
      dr.check_call(run, f'{name} {rng} masked step {k}', ts, call, lanes, device=True)
    dr.compare_streams(run, f'{name} {rng} masked-out lanes', np.flatnonzero(~mask), True)
  _all_reached(f'{name} {rng} masked', run)
  _count(f'masked-{rng}', run)


@pytest.mark.parametrize('rng', ['philox', 'mt19937'])
@pytest.mark.parametrize('name', ['umbrella_d9', 'catch_c9'])
def test_masked_rollout_with_budgets(name, rng):
  T = 8
  run, r = _fresh(name, 512, rng)
  _reset_all(run)
  env = run.env
  mask = r.rand(env.batch) < 0.7
  left = r.randint(0, 3, env.batch).astype(np.int64)
  run.aim_only(np.flatnonzero(mask & (left > 0)))   # the others sit the whole rollout out
  acts = r.randint(0, env.num_actions, (T, env.batch)).astype(np.int32)
  left_oracle = left.copy()
  call = dr.budget_call(acts, mask, left, left_oracle)
  run.inject(call)
  left_dev = torch.from_numpy(left).cuda()
  out = env.make_buffers(T)
  ts = env.rollout(T, actions=torch.from_numpy(acts).cuda(), out=out, mask=torch.from_numpy(mask).cuda(),
                   episodes_left=left_dev)
  dr.check_call(run, f'{name} {rng} masked rollout', ts, call, device=True, t=True)
  assert np.array_equal(left_dev.cpu().numpy(), left_oracle), 'episode budgets'
  _all_reached(f'{name} {rng} masked rollout', run)
  _count(f'masked_rollout-{rng}', run)


# ------------------------------------------------------------------ same-step handles
@pytest.mark.parametrize('final', [True, False], ids=['final_observation', 'no_final_observation'])
@pytest.mark.parametrize('name', ['umbrella_d65', 'umbrella_d129', 'umbrella_d9', 'memory_b33', 'catch'])
def test_same_step(name, final):
  """A LAST and the reset that follows it in one call: umbrella's LAST observation draws its distractors, which the
  final observation replays from the kept stream (final_observation on) or skips (off)."""
  run = dr.run_same_step(name, 'cuda', final, per_class=8, batch=512)
  _count(f'same_step-{final}', run)


# ------------------------------------------------------------------ packs
PACKS = ['catch', 'memory_len', 'umbrella_length', 'mnist', 'cartpole', 'cartpole_swingup', 'mountain_car']


def _pack_run(env, r):
  """Half the lanes aim at a class their setting can reach."""
  labels = np.array(['random'] * env.batch, dtype=object)
  specs = dr.lane_specs(env)
  for i in range(env.batch):
    ok = dr.reachable(specs[i], False)
    if r.rand() < 0.5 and ok:
      labels[i] = ok[r.randint(len(ok))]
  return dr.DrawRun(env, labels, seed=3)


@pytest.mark.parametrize('experiment', PACKS)
def test_packed(experiment, mnist_dir):    # pylint: disable=unused-argument
  """Every setting of the experiment in one handle: lane j of setting k keyed by the setting's seed and lane
  (mnist_dir: the synthetic images the mnist pack loads)."""
  env = bsuite_b200.load_experiment(experiment, 8, device='cuda', seed=21, reward_dtype='float64')
  r = np.random.RandomState(3)
  run = _pack_run(env, r)
  calls = ('reset',) * 2 if experiment in dr.FLOAT_FAMILIES else dr.CALLS
  for k, kind in enumerate(calls):
    if kind == 'reset':
      call = dr.reset_call
    else:
      a = r.randint(0, env.num_actions, env.batch).astype(np.int32)
      call = dr.step_call(a)
    run.inject(call)
    ts = env.reset() if kind == 'reset' else env.step(torch.from_numpy(a).cuda())
    dr.check_call(run, f'pack {experiment} call {k}', ts, call, device=True)
  _all_reached(f'pack {experiment}', run)
  _count('pack', run)


@pytest.mark.parametrize('experiment', ['memory_size', 'umbrella_distract'])
def test_ragged(experiment):
  env = bsuite_b200.load_experiment(experiment, 8, device='cuda', seed=21, reward_dtype='float64', ragged=True)
  r = np.random.RandomState(4)
  run = _pack_run(env, r)
  for k, kind in enumerate(dr.CALLS):
    if kind == 'reset':
      call = dr.reset_call
    else:
      a = r.randint(0, env.num_actions, env.batch).astype(np.int32)
      call = dr.step_call(a)
    run.inject(call)
    ts = env.reset() if kind == 'reset' else env.step(torch.from_numpy(a).cuda())
    dr.check_call(run, f'ragged {experiment} call {k}', ts, call, device=True)
  _all_reached(f'ragged {experiment}', run)
  _count('ragged', run)


# ------------------------------------------------------------------ reduced dtypes, host-driven steps, graphs
@pytest.mark.parametrize('name,obs_dtype', [('catch', 'bfloat16'), ('catch', 'uint8'), ('umbrella_d65', 'bfloat16'),
                                            ('memory_b33', 'bfloat16')])
def test_reduced_obs_dtype(name, obs_dtype):
  run = dr.run_calls(name, 'philox', 'cuda', None, per_class=8, batch=512, obs_dtype=obs_dtype)
  _count(f'obs-{obs_dtype}', run)


@pytest.mark.parametrize('wait', [True, False], ids=['wait', 'no_wait'])
def test_step_host(wait):
  run, r = _fresh('catch', 512)
  _reset_all(run)
  env = run.env
  for k in range(3):
    a = r.randint(0, env.num_actions, env.batch).astype(np.int32)
    call = dr.step_call(a)
    run.inject(call)
    hb = env.make_host_buffers()
    _, dev_obs = env.step_host(torch.from_numpy(a), hb, wait=wait)
    if not wait:
      env.host_wait()
    ts = hb.timestep()
    ts = ts._replace(observation=dev_obs)
    dr.check_call(run, f'step_host wait={wait} call {k}', ts, call, device=True)
  _all_reached(f'step_host wait={wait}', run)
  _count(f'step_host-{wait}', run)


def test_cuda_graph_replay():
  run, r = _fresh('catch', 512)
  _reset_all(run)
  env = run.env
  graphed = env.capture(1)
  a = r.randint(0, env.num_actions, env.batch).astype(np.int32)
  call = dr.step_call(a)
  run.inject(call)                        # after the capture: it restores the state it snapshotted
  graphed.actions.copy_(torch.from_numpy(a)[None].cuda())
  ts = graphed.replay()
  dr.check_call(run, 'graph replay', ts, dr.rollout_call(a[None]), device=True, t=True)
  _all_reached('graph replay', run)
  _count('graph', run)
